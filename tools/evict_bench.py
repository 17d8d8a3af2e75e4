#!/usr/bin/env python
"""What CMB200_EVICT=access costs and buys.

1. Hit ratios: the hot and cold workload of oracle/evict_model.py through the drop-in (cachemap_get, and
   cachemap_put on a miss, then one cold put per step) at --capacity pages of 4 KiB, under CMB200_EVICT=put
   and =access, next to the model's values for the same workload: drawing as the store does
   (model_table) and uniformly (model_uniform).
2. Latency of cmb200_get_small (the method of tools/get_small_bench.py: host clock around calls that
   return when the pages are in page-locked memory, median and p10-p90 microseconds) on an engine without
   the flag and one with CMB200_TOUCH holding the same records, alternated call by call, at 1 and 132
   pages per call and 64 KiB pages.
The card's name and power limit are printed first: they belong beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import edge_fuse_b200 as E
from oracle import evict_model

ap = argparse.ArgumentParser()
ap.add_argument("--capacity", type=int, default=65536, help="pages of the drop-in map")
ap.add_argument("--hot", type=int, default=16384, help="pages of the hot set")
ap.add_argument("--steps", type=int, default=196608)
ap.add_argument("--warmup", type=int, default=131072)
ap.add_argument("--sizes", default="1,132", help="pages per cmb200_get_small call")
ap.add_argument("--reps", type=int, default=200)
ap.add_argument("--skip-ratios", action="store_true")
args = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card}), flush=True)
assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"


def dropin_ratio(policy: str, d: str, seed: int = 1) -> tuple[float, float]:
    """-> (hot-set hit ratio after the warm-up, seconds) of the workload through the drop-in."""
    os.environ["CMB200_EVICT"] = policy
    os.environ["CMB200_PERSIST"] = "0"
    E.binding._libc().srand(seed)
    cm = E.Cachemap(d, args.capacity, 12, 12)
    page = np.zeros(4096, dtype=np.uint8)
    hits = reads = 0
    t0 = time.perf_counter()
    for t in range(args.steps):
        off = (t % args.hot) << 12
        hit = cm.get(off, 1000, 0) is not None
        if not hit:
            cm.put(off, 1000, 0, page)
        cm.put(t << 12, 2000, 0, page)
        if t >= args.warmup:
            reads += 1
            hits += hit
    cm.free()
    return hits / reads, time.perf_counter() - t0


if not args.skip_ratios:
    row = {}
    for policy in ("put", "access"):
        with tempfile.TemporaryDirectory() as d:
            r, s = dropin_ratio(policy, d)
        m = [evict_model.hot_cold(policy == "access", args.capacity, args.hot, args.steps, args.warmup, seed=1,
                                  table=table) for table in (True, False)]
        row[policy] = {"dropin": round(r, 4), "model_table": round(m[0], 4), "model_uniform": round(m[1], 4),
                       "seconds": round(s, 1)}
    print("hit_ratio", json.dumps({"capacity": args.capacity, "hot": args.hot, "steps": args.steps,
                                   "warmup": args.warmup, **row}), flush=True)

# ---- cmb200_get_small latency, flag off and on --------------------------------------------------
PSHIFT = 16
CH = 1 << PSHIFT
sizes = [int(s) for s in args.sizes.split(",")]
n = max(sizes)
GEO = dict(pshift=PSHIFT, accel=12, capacity=1 << 16, arena_bytes=2 << 30, max_batch=1024)
engines = {"off": E.Engine(**GEO), "touch": E.Engine(**GEO, flags=E.TOUCH)}
hp = E.lib().cmb200_host_alloc(n * CH)
try:
    for k, cls in enumerate("RTZM"):
        allc = np.arange(16 * n, dtype=np.uint64)
        cids = allc[((allc + (allc >> np.uint64(3))) & np.uint64(3)) == k][:n]
        pages = np.stack([E.gen_chunk_host(42, int(c), CH) for c in cids])
        u = np.full(n, 100 + k, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        for eng in engines.values():
            eng.put(u, l, pages)
            out, st = eng.get_small(u, l)
            assert (st == E.HIT).all() and (out == pages).all()
        row = {}
        for m in sizes:
            calls = [(f"{w}_n{m}_us", lambda eng=eng, m=m: eng.get_small(u[:m], l[:m], out=hp)) for w, eng in engines.items()]
            t = {name: [] for name, _ in calls}
            for _, fn in calls:
                fn(); fn()
            for _ in range(args.reps):                # off and touch alternate call by call
                for name, fn in calls:
                    t0 = time.perf_counter()
                    fn()
                    t[name].append((time.perf_counter() - t0) * 1e6)
            for name, v in t.items():
                p10, p50, p90 = np.percentile(v, [10, 50, 90])
                row[name] = [round(p50, 1), round(p10, 1), round(p90, 1)]
        print("get_small", cls, json.dumps(row), flush=True)
finally:
    E.lib().cmb200_host_free(hp)
    for eng in engines.values():
        eng.close()
