#!/usr/bin/env python
"""What pinning costs.

1. cmb200_sample: device time of 3 x 4096 draws (one eviction round of ROUND_MAX victims) on an engine of
   --records live 4 KiB records, with 0, 16 and 4096 pin ranges and 0, 25 and 50 % of the live records
   pinned (host clock around the call, which ends in a stream synchronise; median of --reps).
2. cachemap-level calls on one engine: cmb200_pin_count against the list's pages, on both sides of the
   keyed / scan threshold ((cap + 2) / 64 pages), and cmb200_pin_set of 1 and 4096 ranges.
3. Synchronous cachemap_put time at capacity (every put evicts), without pins and with a quarter of the
   capacity pinned: the shape of tools/admit_bench.py.
The card's name and power limit are printed first: they belong beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import edge_fuse_b200 as E
import pin_model as PM

ap = argparse.ArgumentParser()
ap.add_argument("--records", type=int, default=1 << 20)
ap.add_argument("--capacity", type=int, default=65536, help="pages of the drop-in map (part 3)")
ap.add_argument("--puts", type=int, default=20000)
ap.add_argument("--reps", type=int, default=50)
args = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card}), flush=True)
assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e6


def pin_list(n_ranges, frac, n):
    """n_ranges ranges over u = 7 that cover frac of the records 0 .. n-1 (none: ranges of u = 8)."""
    if n_ranges == 0:
        return []
    if frac == 0:
        return [(8, 2 * k, 2 * k) for k in range(n_ranges)]
    per = int(frac * n) // n_ranges
    stride = n // n_ranges
    return [(7, k * stride, k * stride + per - 1) for k in range(n_ranges) if per > 0]


n = args.records
e = E.Engine(pshift=12, capacity=n, arena_bytes=max(256 << 20, n * 128), max_batch=16384)
u = np.full(n, 7, dtype=np.uint64)
for at in range(0, n, 16384):
    m = min(16384, n - at)
    e.put(u[:m], np.arange(at, at + m, dtype=np.uint64), np.zeros((m, 4096), dtype=np.uint8))
r = np.random.default_rng(1).integers(0, 1 << 63, size=3 * 4096, dtype=np.uint64)
for ranges in (0, 16, 4096):
    for frac in (0.0, 0.25, 0.5):
        if ranges == 0 and frac:
            continue
        lst = pin_list(ranges, frac, n)
        e.pin_set(lst)
        us = timed(lambda: e.sample(r), args.reps)
        print(json.dumps({"part": "sample", "ranges": ranges, "pinned": frac, "pages": PM.pages(lst),
                          "us_per_round": round(us, 1)}), flush=True)
cap = e.stats()["table_slots"]
limit = (cap + 2) // 64
for pages in (limit // 4, limit, limit + 1, 4 * limit):
    e.pin_set([(7, 0, pages - 1)])
    us = timed(lambda: e.pin_count(), args.reps)
    print(json.dumps({"part": "pin_count", "pages": pages, "path": "keyed" if pages <= limit else "scan",
                      "table_slots": cap, "us": round(us, 1)}), flush=True)
for k in (1, 4096):
    lst = [(7, 2 * i, 2 * i) for i in range(k)]
    us = timed(lambda: e.pin_set(lst), args.reps)
    print(json.dumps({"part": "pin_set", "ranges": k, "us": round(us, 1)}), flush=True)
e.close()

os.environ.update(CMB200_PERSIST="0", CMB200_WB_SLOTS="0")
for k in ("CMB200_ADMIT", "CMB200_EVICT", "CMB200_GHOST", "CMB200_HOST_TIER_MB", "CMB200_DEVICES"):
    os.environ.pop(k, None)
page = np.zeros(4096, dtype=np.uint8)
for pinned in (0, args.capacity // 4):
    with tempfile.TemporaryDirectory() as d:
        cm = E.Cachemap(d, args.capacity, 12, 12)
        if pinned:
            assert cm.pin(1, 0, 0, pinned * 4096) == pinned
        for p in range(args.capacity):
            cm.put(p << 12, 1, 0, page)
        t = []
        for p in range(args.capacity, args.capacity + args.puts):
            page[:8] = np.frombuffer(np.uint64(p).tobytes(), dtype=np.uint8)
            t0 = time.perf_counter()
            cm.put(p << 12, 1, 0, page)
            t.append(time.perf_counter() - t0)
        print(json.dumps({"part": "put_at_capacity", "pinned": pinned, "median_us": round(float(np.median(t)) * 1e6, 1),
                          "p90_us": round(float(np.percentile(t, 90)) * 1e6, 1),
                          "pin_stats": cm.pin_stats()}), flush=True)
        cm.free()
