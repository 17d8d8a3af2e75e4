#!/usr/bin/env python
"""Latency of the fused small-batch get (cmb200_get_small) per content class and batch size, next to
the two-kernel batch path (cmb200_get_batch) on the same requests.  Tuning aid."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import edge_fuse_b200 as E

CH = 65536
n = 256
eng = E.Engine(pshift=16, accel=12, capacity=1 << 16, arena_bytes=2 << 30, max_batch=1024)
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
    for m in (1, 8, 32, 132, 256):
        for name, fn in (("small", lambda: eng.get_small(u[:m], l[:m], out=hp)), ("batch", lambda: eng.get(u[:m], l[:m], out=hp))):
            fn(); fn()
            reps = 20
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            dt = (time.perf_counter() - t0) / reps
            row[f"{name}_n{m}_us"] = round(dt * 1e6, 1)
    res[cls] = row
    print(cls, json.dumps(row), flush=True)
eng.close()
