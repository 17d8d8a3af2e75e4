#!/usr/bin/env python
"""What rebuilding parse checkpoints costs cmb200_load: wall time of loading one snapshot of T and M
pages (text-like, and text repeated: the classes with the most sequences per page) into a fresh
engine with the checkpoint side table and into one created with CMB200_CKPT=0, alternated.  The
snapshot is written to a temporary directory and read once before the timed loads, so that they find
it in the page cache.  --profile instead loads it once under torch.profiler and reports the kernel
time of k_restore (the kernel that copies the records in and walks their blocks) in both engines."""
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
ap.add_argument("--gib", type=float, default=4.0, help="snapshot size to reach (record bytes)")
ap.add_argument("--pshift", type=int, default=16)
ap.add_argument("--runs", type=int, default=3, help="loads of each kind, alternated")
ap.add_argument("--profile", action="store_true")
args = ap.parse_args()

CH = 1 << args.pshift
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card, "pshift": args.pshift, "target_gib": args.gib}), flush=True)
arena = int(args.gib * 1.5 * (1 << 30)) + (1 << 30)
GEO = dict(pshift=args.pshift, accel=12, capacity=1 << 20, arena_bytes=arena, max_batch=1024)


def engine(ckpt: bool):
    if ckpt:
        return E.Engine(**GEO)
    os.environ["CMB200_CKPT"] = "0"
    try:
        return E.Engine(**GEO)
    finally:
        del os.environ["CMB200_CKPT"]


with tempfile.TemporaryDirectory() as tmp:
    path = os.path.join(tmp, "big.snap")
    src = engine(True)
    B = 1024
    dev = src.dev_alloc(B * CH)
    # T (class 1) and M (class 3) chunks of the synthetic stream
    allc = np.arange(1 << 20, dtype=np.uint64)
    cls = (allc + (allc >> np.uint64(3))) & np.uint64(3)
    cids = allc[(cls == 1) | (cls == 3)]
    put = 0
    while src.stats()["arena_used"] < args.gib * (1 << 30):
        c = cids[put:put + B]
        src.gen_chunks_dev(42, c, dev)
        src.put(np.full(B, 7, dtype=np.uint64), np.arange(put, put + B, dtype=np.uint64), dev, on_dev=True)
        put += B
    src.dev_free(dev)
    records = src.save(path)
    src.close()
    size = os.path.getsize(path)
    with open(path, "rb") as f:                        # into the page cache
        while f.read(64 << 20):
            pass
    print(json.dumps({"records": records, "snapshot_bytes": size}), flush=True)

    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        for name in ("ckpt", "nockpt"):
            eng = engine(name == "ckpt")
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                eng.load(path)
            eng.close()
            k = [e for e in prof.events() if e.device_type.name == "CUDA" and "k_restore" in e.name]
            us = sum(e.time_range.end - e.time_range.start for e in k)
            print(json.dumps({"engine": name, "k_restore_launches": len(k), "k_restore_ms": round(us / 1e3, 2),
                              "per_record_us": round(us / max(1, records), 3)}), flush=True)
    else:
        res = {"ckpt": [], "nockpt": []}
        for r in range(args.runs):
            for name in ("ckpt", "nockpt"):
                eng = engine(name == "ckpt")
                t0 = time.perf_counter()
                got = eng.load(path)
                dt = time.perf_counter() - t0
                assert got == records
                if r == 0:
                    _, ok = eng.read_checkpoints(np.full(min(records, 4096), 7, dtype=np.uint64),
                                                 np.arange(min(records, 4096), dtype=np.uint64))
                    res[f"{name}_with_checkpoints"] = round(float((ok == 1).mean()), 3)
                eng.close()
                res[name].append(round(dt, 3))
                print(name, round(dt, 3), "s", round(size / dt / (1 << 30), 2), "GiB/s", flush=True)
        print(json.dumps(res), flush=True)
