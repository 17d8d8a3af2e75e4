"""Cost of cmb200_rename against what a caller could do without it, and of the drop-in's rename.

Engine, pshift 12 (4 KiB) and 16 (64 KiB) pages, n = 1, 16, 256, 4096 and 16384 pages per call, all of
one class of the synthetic stream (R: random bytes, T: text-like), two ways of moving n cached pages of
one object to another, alternated in one loop, each call timed by a host clock that ends in a
synchronise of the engine's stream:
- rename: one cmb200_rename of the n pages;
- copy:   cmb200_get_batch of the old name into page-locked memory, cmb200_put_batch at the new name
          (every page encoded again), cmb200_invalidate of the old name.
The pages go back and forth between two names, so the store keeps its size; the arena is compacted
between rounds (untimed) when half of it is used.  Median and p10-p90 in microseconds per call.

Drop-in, on one engine with the write-behind ring off, a 64 MiB file of T pages at 64 KiB pages (1 024
pages) and a 64 MiB file of T pages at 4 KiB pages (16 384 pages):
- cachemap_rename of the file, then the first cachemap_read_range of the new name (all hits);
- the same with the two invalidations that replace it (cachemap_invalidate of both names), then the
  first read_range, which misses on its first page; the refill from the edge server cannot be measured
  here, so the GPU part of it, cachemap_write_range of the file (every page encoded again), is timed
  on its own.
The card's name and power limit are read in the same run.  One JSON line per measurement.

usage: python tools/rename_bench.py [--reps 15] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import edge_fuse_b200 as E  # noqa: E402

KINDS = {"R": 0, "T": 1}          # content class of the synthetic stream: 0 random bytes, 1 text-like
TO_END = (1 << 64) - 1


def stream_class(cid):
    """The class of chunk cid (sg_class, edge_fuse_b200/csrc/streamgen.cuh)."""
    return (cid + (cid >> 3)) & 3


def class_pages(kind, n, bs):
    cids = [c for c in range(8 * n + 8) if stream_class(c) == KINDS[kind]][:n]
    return np.stack([E.gen_chunk_host(11, c, bs) for c in cids])


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def summary(ts):
    us = np.array(ts) * 1e6
    return {"median_us": round(float(np.median(us)), 1), "p10_us": round(float(np.percentile(us, 10)), 1),
            "p90_us": round(float(np.percentile(us, 90)), 1), "calls": len(us)}


def engine_run(lib, eng, kind, n, reps, warmup):
    bs = eng.bsize
    pages = class_pages(kind, n, bs)
    names = (2000 + KINDS[kind], 3000 + KINDS[kind])
    l = np.arange(n, dtype=np.uint64)
    eng.put(np.full(n, names[0], dtype=np.uint64), l, pages)
    addr = [np.ascontiguousarray(np.stack([np.full(n, u, dtype=np.uint64), l], axis=1)) for u in names]
    status = np.zeros(n, dtype=np.int32)
    host = lib.cmb200_host_alloc(n * bs)
    t_ren, t_copy = [], []
    try:
        at = 0                                        # the name that holds the pages
        for i in range(warmup + reps):
            for how in ("rename", "copy"):
                st = eng.stats()
                if st["arena_used"] > st["arena_bytes"] // 2:
                    eng.compact()
                src, dst = names[at], names[1 - at]
                t0 = time.perf_counter()
                if how == "rename":
                    moved = eng.rename(src, dst, 0, n - 1)
                    ok = moved == (n, 0)
                else:
                    rc = lib.cmb200_get_batch(eng.h, n, addr[at].ctypes.data, None, host, status.ctypes.data)
                    ok = rc == 0 and (status == E.HIT).all()
                    rc = lib.cmb200_put_batch(eng.h, n, addr[1 - at].ctypes.data, None, host, None, None)
                    ok = ok and rc == 0 and eng.invalidate(src, 0, n - 1) == n
                t1 = time.perf_counter()
                if not ok:
                    raise RuntimeError(f"{how}: {E.last_error()}")
                at = 1 - at
                if i >= warmup:
                    (t_ren if how == "rename" else t_copy).append(t1 - t0)
        got, gs = eng.get(np.full(n, names[at], dtype=np.uint64), l)
        if not ((gs == E.HIT).all() and (got == pages).all()):
            raise RuntimeError("the pages read back differ")
        eng.invalidate(names[at], 0, TO_END)
    finally:
        lib.cmb200_host_free(host)
    return {"rename": summary(t_ren), "copy": summary(t_copy)}


def drop_in_run(pshift, reps):
    bs = 1 << pshift
    n = (64 << 20) // bs
    data = class_pages("T", n, bs).tobytes()
    os.environ.update(CMB200_WB_SLOTS="0", CMB200_PERSIST="0")
    res = {"rename": [], "read_after_rename": [], "invalidate_both": [], "read_after_invalidate": [],
           "refill_put": []}
    with tempfile.TemporaryDirectory() as d:
        cm = E.Cachemap(d, 1 << 18, 12, pshift)     # an arena with room for both files and their garbage
        try:
            for i in range(reps + 1):
                cm.write_range(10, 0, 0, data)       # f.tmp
                cm.write_range(11, 0, 0, data)       # f, replaced
                if cm.read_range(10, 0, 0, len(data)) is None:
                    raise RuntimeError("the written file is not cached whole")
                drops = sum(E.engine_stats(h)["dropped_puts"] for h in cm.engine_handles())
                t0 = time.perf_counter()
                moved = cm.rename(10, 11, 0)
                t1 = time.perf_counter()
                got = cm.read_range(11, 0, 0, len(data))
                t2 = time.perf_counter()
                if moved != n or got is None or bytes(got) != data:
                    drops = sum(E.engine_stats(h)["dropped_puts"] for h in cm.engine_handles()) - drops
                    raise RuntimeError(f"drop-in rename: moved {moved} of {n}, dropped {drops}")
                cm.write_range(10, 0, 0, data)
                t3 = time.perf_counter()
                cm.invalidate(11, 0, 0, E.Cachemap.TO_END)
                cm.invalidate(10, 0, 0, E.Cachemap.TO_END)
                t4 = time.perf_counter()
                miss = cm.read_range(11, 0, 0, len(data))
                t5 = time.perf_counter()
                cm.write_range(11, 0, 0, data)       # the refill's put, once the server has sent the bytes
                t6 = time.perf_counter()
                if miss is not None:
                    raise RuntimeError("an invalidated file was served")
                if i:
                    for k, v in zip(res, (t1 - t0, t2 - t1, t4 - t3, t5 - t4, t6 - t5)):
                        res[k].append(v)
                cm.invalidate(11, 0, 0, E.Cachemap.TO_END)
        finally:
            cm.free()
    return {k: summary(v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if E.device_count() < 1:
        raise SystemExit(f"no CUDA device: {E.last_error()}")
    lib = E.lib()
    dev = card()
    for pshift in (12, 16):
        eng = E.Engine(pshift=pshift, accel=12, capacity=65536, arena_bytes=6 << 30, max_batch=4096)
        try:
            for kind in KINDS:
                for n in (1, 16, 256, 4096, 16384):
                    r = engine_run(lib, eng, kind, n, a.reps, a.warmup)
                    print(json.dumps({"tool": "rename_bench", "card": dev, "pages": kind, "page_bytes": 1 << pshift,
                                      "pages_per_call": n, **r}), flush=True)
        finally:
            eng.close()
    for pshift in (16, 12):
        r = drop_in_run(pshift, max(3, a.reps // 3))
        print(json.dumps({"tool": "rename_bench", "card": dev, "drop_in": f"64 MiB file, T pages, {1 << pshift >> 10} KiB pages",
                          "pages": (64 << 20) >> pshift, **r}), flush=True)


if __name__ == "__main__":
    main()
