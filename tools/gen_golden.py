#!/usr/bin/env python
"""Generates tests/golden/*.json from the reference itself (oracle/_ref/libcachemap_ref.so, i.e.
/root/reference/cachemap compiled unmodified, plus oracle/ref_kat.c built against the reference's
own uint128.h).  Run in the authoring container only; the fixtures it writes are committed and
are what pins the oracle (and, on the GPU box, the CUDA path) where /root/reference is absent.

    python tools/gen_golden.py [lz4 keys ref_blocks limit exerciser store]
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import datagen  # noqa: E402
from oracle import ef_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
REF = "/root/reference/cachemap"


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def gen_lz4():
    out = []
    for kind, n, accel, seed in datagen.codec_cases():
        page = datagen.make_page(kind, n, seed)
        blk = O.ref_lz4_encode(page, accel)
        rec = {"kind": kind, "n": n, "accel": accel, "seed": seed, "in_sha256": sha(page),
               "len": len(blk), "sha256": sha(blk)}
        if len(blk) <= 300:
            rec["hex"] = blk.hex()
        if n:
            back, used = O.ref_lz4_decode(blk, n)
            assert back == page.tobytes() and used == len(blk)
        out.append(rec)
    with open(os.path.join(GOLD, "lz4_blocks.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast of cachemap/lz4.c (v1.8.1), "
                   "called as filemap.c:126 does", "cases": out}, f, indent=0)
    print("lz4 cases:", len(out))


def gen_ref_blocks():
    """Length and SHA-256 of the reference's block for every page of the oracle's sweep and of the
    CUDA comparison, so that both comparisons run without the reference."""
    def rows(cases):
        out = []
        for kind, n, accel, seed in cases:
            page = datagen.make_page(kind, n, seed)
            blk = O.ref_lz4_encode(page, accel)
            back, used = O.ref_lz4_decode(blk, n)
            assert back == page.tobytes() and used == len(blk)
            out.append([kind, n, accel, seed, len(blk), sha(blk)[:32]])
        return out
    with open(os.path.join(GOLD, "ref_blocks.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast of cachemap/lz4.c (v1.8.1)",
                   "version": O.ref().LZ4_versionString().decode(),
                   "columns": ["kind", "n", "accel", "seed", "len", "sha256 (first 32 hex digits)"],
                   "sweep": rows(datagen.reference_sweep_cases()),
                   "gpu": rows(datagen.gpu_reference_cases())}, f, indent=0)
    print("reference blocks written")


def gen_limit():
    """The reference's LZ4_compress_fast with filemap_set's dstCapacity of n + 1024 (filemap.c:126) on
    pages whose unlimited block is within 24 bytes of that limit (pshift 18-20), plus random pages at
    pshift 17, where every block fits.  ref_len 0: the reference refused the page."""
    out = []
    for pshift in (17, 18, 19, 20):
        n = 1 << pshift
        for seed in range(3):
            for accel in (12, 1):
                base = len(O.lz4_encode(datagen.limit_page(n, 100 * pshift + seed, 0, 0), accel))
                # a zero run near the page start (where the match search still steps byte by byte)
                # shortens the block by about its length
                zlens = [0] if pshift == 17 else range(max(0, base - n - 1024 - 24), base - n - 1024 + 25, 2)
                for z in zlens:
                    at = 16 * seed
                    page = datagen.limit_page(n, 100 * pshift + seed, at, z)
                    ours = len(O.lz4_encode(page, accel))
                    if pshift > 17 and abs(ours - (n + 1024)) > 24:
                        continue
                    out.append([pshift, accel, 100 * pshift + seed, at, z, len(O.ref_lz4_encode(page, accel))])
    with open(os.path.join(GOLD, "lz4_limit.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast(page, dst, n, n + 1024, accel) "
                   "of cachemap/lz4.c (v1.8.1), called as filemap.c:126 does",
                   "columns": ["pshift", "accel", "seed", "zero_at", "zero_len", "ref_len (0: refused)"],
                   "page": "tests/datagen.py limit_page(1 << pshift, seed, zero_at, zero_len)", "cases": out}, f, indent=0)
    print("limit cases:", len(out), "refused:", sum(1 for r in out if r[-1] == 0))


def gen_exerciser(seeds=(1, 2, 3), objects=32768, pshift=15):
    """Per-phase hit counts of tests/c/exerciser.c linked against the reference's library."""
    import re
    ref = os.path.join(ROOT, "oracle", "_ref", "libcachemap_ref.so")
    exe = os.path.join(ROOT, "oracle", "_ref", "exerciser_ref")
    subprocess.run(["gcc", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c", "exerciser.c"),
                    "-o", exe, ref, f"-Wl,-rpath,{os.path.dirname(ref)}", "-lpthread"], check=True)
    runs = []
    for seed in seeds:
        for attempt in range(8):                   # the reference can hang at start-up (SURVEY.md §5)
            with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
                try:
                    out = subprocess.run([exe, d, str(objects), str(pshift), str(seed)], capture_output=True,
                                         text=True, timeout=60).stdout
                    break
                except subprocess.TimeoutExpired:
                    continue
        else:
            raise RuntimeError("the reference exerciser hung at start-up in every attempt")
        phases = {m.group(1): [int(m.group(2)), int(m.group(3))] for m in re.finditer(r"phase (\w+) hits (\d+) of (\d+)", out)}
        entries = [int(x) for x in re.findall(r"entries_after_\w+ (\d+)", out)]
        assert len(phases) == 5, out
        runs.append({"seed": seed, "phases": phases, "entries": entries})
    with open(os.path.join(GOLD, "ref_exerciser.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py: tests/c/exerciser.c linked against libcachemap_ref.so (LMDB on tmpfs)",
                   "objects": objects, "pshift": pshift, "runs": runs}, f, indent=1)
    print("exerciser runs:", runs)


def gen_keys():
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_kat")
    subprocess.run(["gcc", "-O2", "-I" + REF, os.path.join(ROOT, "oracle", "ref_kat.c"), "-o", exe], check=True)
    data = json.loads(subprocess.run([exe], check=True, capture_output=True, text=True).stdout)
    data["generator"] = "oracle/ref_kat.c compiled against the reference's cachemap/uint128.h"
    with open(os.path.join(GOLD, "keys.json"), "w") as f:
        json.dump(data, f, indent=0)
    print("key KATs:", len(data["addrs"]))


def store_script(pshift=16):
    """The operation list of the store trace: C0 shape (16 x 64 KiB) plus the edge cases of
    SURVEY.md §8c.  Each op: [kind, offset, nhid, genid, content]; content = [kind, seed]."""
    import edge_fuse_b200 as E
    ops = []
    cids = list(range(16))
    off, nh = E.gen_addr(42, cids, pshift)
    for c in cids:                                   # 16 puts, config 0
        ops.append(["put", int(off[c]), int(nh[c]), 0, ["S", c]])
    for c in cids:
        ops.append(["get", int(off[c]), int(nh[c]), 0, None])
    ops.append(["put", 16 << pshift, int(nh[0]), 0, ["S", 3]])        # same content, new address
    ops.append(["get", 16 << pshift, int(nh[0]), 0, None])
    ops.append(["put", int(off[5]), int(nh[5]), 0, ["T", 999]])       # same address, new content
    ops.append(["get", int(off[5]), int(nh[5]), 0, None])
    ops.append(["get", 40 << pshift, int(nh[0]), 0, None])            # never stored
    ops.append(["get", (1 << pshift) + 1, int(nh[1]), 0, None])       # offset truncated by >> pshift
    ops.append(["get", int(off[2]), int(nh[2]), 7, None])             # other genid: miss
    ops.append(["put", int(off[2]), int(nh[2]), 7, ["Z", 5]])
    ops.append(["get", int(off[2]), int(nh[2]), 7, None])
    ops.append(["get", int(off[2]), int(nh[2]), 0, None])
    ops.append(["put", (1 << 44) << pshift, 1, 0, ["R", 1]])          # page number overflows 44 bits
    ops.append(["get", (1 << 44) << pshift, 1, 0, None])
    ops.append(["get", int(off[2]), int(nh[2]), (1 << 20) + 7, None]) # genid keeps its low 20 bits only
    ops.append(["put", int(off[9]), int(nh[9]), 0, ["R", 77]])
    ops.append(["put", int(off[9]), int(nh[9]), 0, ["M", 78]])        # twice in a row: last wins
    ops.append(["get", int(off[9]), int(nh[9]), 0, None])
    return ops


def gen_store():
    R = O.ref()
    pshift, accel = 16, 12
    ops = store_script(pshift)
    trace = []
    with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
        assert not R.cachemap_create(d.encode(), 1023, accel, pshift)         # n < 1024 -> NULL
        assert not R.cachemap_create((d + "/nope").encode(), 1024, accel, pshift)
        cm = R.cachemap_create(d.encode(), 1024, accel, pshift)
        assert cm
        libc = C.CDLL(None)
        libc.free.argtypes = [C.c_void_p]
        for kind, off, nh, gen, content in ops:
            if kind == "put":
                page = datagen.make_page(content[0], 1 << pshift, content[1])
                R.cachemap_put(cm, off, nh, gen, page.ctypes.data)
                trace.append(None)
            else:
                p = R.cachemap_get(cm, off, nh, gen)
                if p:
                    trace.append(sha(C.string_at(p, 1 << pshift)))
                    libc.free(p)
                else:
                    trace.append("miss")
        pages_ptr = C.cast(cm, C.POINTER(C.c_void_p))[0]                      # cm->pages
        entries = int(R.filemap_entries(pages_ptr))
        # struct cachemap tail: capacity, requests, hits are its last three u64 (cachemap.h:20-31)
        sz = 8 + 8 + 8 + 4 * 8 + 48 + 40 + 8 + 3 * 8
        raw = C.string_at(cm, sz)
        cap, req, hits = np.frombuffer(raw[-24:], dtype=np.uint64)
        assert cap == 1024, cap
        # deliberately no cachemap_free(): it can hang in the reference (SURVEY.md §5)
    with open(os.path.join(GOLD, "store_trace.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py against libcachemap_ref.so (LMDB on tmpfs)",
                   "pshift": pshift, "accel": accel, "capacity": 1024, "ops": ops, "gets": trace,
                   "entries": entries, "requests": int(req), "hits": int(hits),
                   "create_null": ["capacity 1023", "missing directory"]}, f, indent=0)
    print("store trace ops:", len(ops), "entries", entries, "requests", int(req), "hits", int(hits))
    os._exit(0)


if __name__ == "__main__":
    assert O.ref() is not None, "oracle/_ref/libcachemap_ref.so missing: run make -C oracle"
    os.makedirs(GOLD, exist_ok=True)
    steps = {"lz4": gen_lz4, "keys": gen_keys, "ref_blocks": gen_ref_blocks, "limit": gen_limit, "exerciser": gen_exerciser,
             "store": gen_store}                   # gen_store ends the process: keep it last
    for name in sys.argv[1:] or steps:
        steps[name]()
