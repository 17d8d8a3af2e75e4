#!/usr/bin/env python
"""Latency of the fused small-batch get (cmb200_get_small) per content class and batch size, next to
the two-kernel batch path (cmb200_get_batch, on the first way's engine) on the same requests: median
and p10-p90 microseconds per call.  --pshift 17 measures the two-CTA cluster decoder of 128 KiB
pages.  Tuning aid.

--ways names how the records reach the store, each into an engine of its own, measured alternately:
fresh (puts: the encoder's parse checkpoints), load (save + load: checkpoints rebuilt from the block),
compact (the records moved down by a compaction after 10 % of the keys were unset), nockpt (puts
into an engine created with CMB200_CKPT=0: every record is parsed by one warp)."""
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

ap = argparse.ArgumentParser()
ap.add_argument("--pshift", type=int, default=16)
ap.add_argument("--sizes", default="1,8,32,132,256", help="pages per call")
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--ways", default="fresh", help="comma list of fresh, load, compact, nockpt")
args = ap.parse_args()

CH = 1 << args.pshift
sizes = [int(s) for s in args.sizes.split(",")]
ways = args.ways.split(",")
n = max(sizes)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card, "pshift": args.pshift, "ways": ways}), flush=True)
GEO = dict(pshift=args.pshift, accel=12, capacity=1 << 16, arena_bytes=2 << 30, max_batch=1024)


def engine(way):
    if way != "nockpt":
        return E.Engine(**GEO)
    os.environ["CMB200_CKPT"] = "0"
    try:
        return E.Engine(**GEO)
    finally:
        del os.environ["CMB200_CKPT"]


def store(eng, way, u, l, pages, tmp):
    """Puts the pages into eng the way `way` names."""
    if way == "load":
        src = E.Engine(**GEO)
        src.put(u, l, pages)
        path = os.path.join(tmp, "w.snap")
        src.save(path)
        src.close()
        eng.load(path)
    elif way == "compact":
        extra = max(1, len(u) // 9)                   # 10 % of the keys, put first and unset
        eu = np.full(extra, 99, dtype=np.uint64); el = np.arange(extra, dtype=np.uint64)
        eng.put(eu, el, pages[:extra])
        eng.put(u, l, pages)
        eng.unset(eu, el)
        eng.compact()
    else:
        eng.put(u, l, pages)


engines = {w: engine(w) for w in ways}
hp = E.lib().cmb200_host_alloc(n * CH)
res = {}
with tempfile.TemporaryDirectory() as tmp:
    for k, cls in enumerate("RTZM"):
        allc = np.arange(16 * n, dtype=np.uint64)
        cids = allc[((allc + (allc >> np.uint64(3))) & np.uint64(3)) == k][:n]
        pages = np.stack([E.gen_chunk_host(42, int(c), CH) for c in cids])
        u = np.full(n, 100 + k, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
        row = {}
        for w, eng in engines.items():
            store(eng, w, u, l, pages, tmp)
            out, st = eng.get_small(u, l)
            assert (st == E.HIT).all() and (out == pages).all()
            _, ok = eng.read_checkpoints(u, l)
            row[f"ckpt_{w}"] = round(float((ok == 1).mean()), 3)   # share of records with checkpoints
        for m in sizes:
            calls = [(f"small_n{m}_us" if w == "fresh" else f"small_{w}_n{m}_us",
                      lambda eng=eng: eng.get_small(u[:m], l[:m], out=hp)) for w, eng in engines.items()]
            eng0 = next(iter(engines.values()))
            calls.append((f"batch_n{m}_us", lambda: eng0.get(u[:m], l[:m], out=hp)))
            t = {name: [] for name, _ in calls}
            for _, fn in calls:
                fn(); fn()
            for _ in range(args.reps):                # the ways alternate call by call
                for name, fn in calls:
                    t0 = time.perf_counter()
                    fn()                               # both calls return after the pages are in `hp`
                    t[name].append((time.perf_counter() - t0) * 1e6)
            for name, v in t.items():
                p10, p50, p90 = np.percentile(v, [10, 50, 90])
                row[name] = [round(p50, 1), round(p10, 1), round(p90, 1)]
        res[cls] = row
        print(cls, json.dumps(row), flush=True)
E.lib().cmb200_host_free(hp)
for eng in engines.values():
    eng.close()
