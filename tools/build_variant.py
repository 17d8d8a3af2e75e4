#!/usr/bin/env python
"""Builds a variant of libcachemap.so.0.0 with extra -D flags into
edge_fuse_b200/build/variants/<name>.so (select it with CMB200_LIB=<path>), e.g. the encoder
timeline build that tools/encode_timeline.py reads:

    python tools/build_variant.py timeline -DCMB_ENC_TIMELINE
"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from edge_fuse_b200 import build as B

name, defs = sys.argv[1], sys.argv[2:]
out_dir = os.path.join(B.OBJ, "variants")
os.makedirs(out_dir, exist_ok=True)
nvcc = B._nvcc()
objs = []
for src in B.CU_SOURCES:
    obj = os.path.join(out_dir, f"{name}_{src[:-3]}.o")
    subprocess.run([nvcc, *B.NVCC_FLAGS, *defs, "-c", os.path.join(B.CSRC, src), "-o", obj], check=True)
    objs.append(obj)
objs.append(os.path.join(B.OBJ, "cachemap_api.o"))
out = os.path.join(out_dir, f"{name}.so")
subprocess.run([nvcc, "-shared", *B.GENCODE, "-o", out, *objs,
                "-Xlinker", "-soname=libcachemap.so.0.0", "-lpthread"], check=True)
print(out)
