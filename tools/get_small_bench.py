#!/usr/bin/env python
"""Latency of the fused small-batch get (cmb200_get_small) per content class and batch size, next to
the two-kernel batch path (cmb200_get_batch) on the same requests: median and p10-p90 microseconds
per call.  --pshift 17 measures the two-CTA cluster decoder of 128 KiB pages.  Tuning aid."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import edge_fuse_b200 as E

ap = argparse.ArgumentParser()
ap.add_argument("--pshift", type=int, default=16)
ap.add_argument("--sizes", default="1,8,32,132,256", help="pages per call")
ap.add_argument("--reps", type=int, default=50)
args = ap.parse_args()

CH = 1 << args.pshift
sizes = [int(s) for s in args.sizes.split(",")]
n = max(sizes)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card, "pshift": args.pshift}), flush=True)
eng = E.Engine(pshift=args.pshift, accel=12, capacity=1 << 16, arena_bytes=2 << 30, max_batch=1024)
hp = E.lib().cmb200_host_alloc(n * CH)
res = {}
for k, cls in enumerate("RTZM"):
    allc = np.arange(16 * n, dtype=np.uint64)
    cids = allc[((allc + (allc >> np.uint64(3))) & np.uint64(3)) == k][:n]
    pages = np.stack([E.gen_chunk_host(42, int(c), CH) for c in cids])
    u = np.full(n, 100 + k, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
    eng.put(u, l, pages)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    row = {}
    for m in sizes:
        for name, fn in (("small", lambda: eng.get_small(u[:m], l[:m], out=hp)), ("batch", lambda: eng.get(u[:m], l[:m], out=hp))):
            fn(); fn()
            t = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                fn()                                   # both calls return after the pages are in `hp`
                t.append((time.perf_counter() - t0) * 1e6)
            p10, p50, p90 = np.percentile(t, [10, 50, 90])
            row[f"{name}_n{m}_us"] = [round(p50, 1), round(p10, 1), round(p90, 1)]
    res[cls] = row
    print(cls, json.dumps(row), flush=True)
E.lib().cmb200_host_free(hp)
eng.close()
