"""Builds libcachemap.so.0.0 (CUDA kernels + engine + C API) in-tree for sm_90a (H100).

nvcc cross-compiles without a GPU; the resulting shared object is git-ignored but travels to the
GPU box with the repo snapshot.  Usage: ``python -m edge_fuse_b200.build`` or ``build()``.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libcachemap.so.0.0")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper)
NVCC_FLAGS = [
    *GENCODE, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xcompiler", "-Wno-unknown-pragmas",
]
CU_SOURCES = ["kernels.cu", "engine.cu"]
C_SOURCES = ["cachemap_api.c"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the cachemap library cannot be built (no CPU fallback exists)")


def _newer(src_paths, target) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(p) > t for p in src_paths)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps += [os.path.join(HERE, "..", "include", f) for f in os.listdir(os.path.join(HERE, "..", "include"))]
    if not force and not _newer(deps, LIB):
        return LIB
    nvcc = _nvcc()
    objs = []
    for src in CU_SOURCES:
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.run(cmd, check=True)
        objs.append(obj)
    for src in C_SOURCES:
        obj = os.path.join(OBJ, src.replace(".c", ".o"))
        subprocess.run(["gcc", "-std=gnu11", "-O2", "-fPIC", "-Wall", "-Wextra", "-pthread", "-c",
                        os.path.join(CSRC, src), "-o", obj], check=True)
        objs.append(obj)
    subprocess.run([nvcc, "-shared", *GENCODE, "-o", LIB, *objs,
                    "-Xlinker", "-soname=libcachemap.so.0.0", "-lpthread"], check=True)
    link = os.path.join(HERE, "libcachemap.so")
    if os.path.lexists(link):
        os.remove(link)
    os.symlink("libcachemap.so.0.0", link)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
