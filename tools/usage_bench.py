#!/usr/bin/env python
"""What the usage and residency calls cost.

1. cmb200_residency on engines of 2^22 and 2^27 table slots holding --records live 4 KiB records: keyed at
   1, 16 and 1024 pages and a whole-object scan (every page number of one genid), host clock around the
   call, which ends in a stream synchronise; median of --reps.  Whether invalidation's keyed / scan
   threshold ((cap + 2) / 64 addresses) suits residency shows in the keyed time at the threshold against
   the scan time, printed as well.
2. cmb200_usage_set over one engine of about 2^20 and 2^25 live 4 KiB records, with 1, 16 and 256 pages per
   object: call time (median of --usage-reps) and the peak scratch HBM (the lowest free device memory seen by
   a thread polling cudaMemGetInfo during the calls, against the free memory before them).
3. cachemap_get p50 / p99 from 8 and 32 native threads (tools/usage_serve.c), idle and while another
   thread calls cachemap_usage back to back.
The card's name and power limit are printed first: they belong beside the numbers.  Scratch files go to a
temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import edge_fuse_b200 as E

ap = argparse.ArgumentParser()
ap.add_argument("--records", type=int, default=1 << 20, help="live records of part 1's engines")
ap.add_argument("--usage-records", default=f"{1 << 20},{1 << 25}")
ap.add_argument("--per-object", default="1,16,256")
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--usage-reps", type=int, default=5)
ap.add_argument("--serve-pages", type=int, default=1 << 18)
ap.add_argument("--serve-gets", type=int, default=4000)
ap.add_argument("--skip", default="", help="comma-separated parts to skip (1, 2, 3)")
args = ap.parse_args()
skip = set(args.skip.split(",")) - {""}

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card}), flush=True)
assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"
STEP = 1 << 16


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e6


def filled(slots, n, per_object, arena):
    """An engine of `slots` table slots with n records of 4 KiB, per_object consecutive pages per object
    (u = 1000 + record // per_object), the pages on the device."""
    e = E.Engine(pshift=12, capacity=n, arena_bytes=arena, table_slots=slots, max_batch=STEP)
    dev = e.dev_alloc(STEP * 4096)
    e.h2d(dev, np.zeros((STEP, 4096), dtype=np.uint8))
    for at in range(0, n, STEP):
        m = min(STEP, n - at)
        k = np.arange(at, at + m, dtype=np.uint64)
        e.put(np.uint64(1000) + k // np.uint64(per_object), k % np.uint64(per_object), dev, on_dev=True)
    e.sync()
    e.dev_free(dev)
    assert e.stats()["entries"] == n, e.stats()
    return e


# ---- 1. residency --------------------------------------------------------------------------------------------
if "1" not in skip:
    n = args.records
    for slots in (1 << 22, 1 << 27):
        e = filled(slots, n, 2048, 256 << 20)
        limit = (slots + 2) // 64
        u = 1000 + n // 2048 // 2
        for pages in (1, 16, 1024, limit):
            us = timed(lambda: e.residency(u, 0, pages - 1), args.reps)
            print(json.dumps({"part": "residency", "table_slots": slots, "path": "keyed", "pages": pages,
                              "us": round(us, 1)}), flush=True)
        us = timed(lambda: e.residency(u, 0, limit), args.reps)
        print(json.dumps({"part": "residency", "table_slots": slots, "path": "scan", "pages": limit + 1,
                          "us": round(us, 1)}), flush=True)
        # a whole object: every page number of genid 0 (2^44 addresses), found by the scan.  The engine call
        # writes only the bytes of the records it finds, all below page 2048 here, so a 4 KiB vector holds them.
        got = e.residency(u, 0, 4095)
        assert int((got == 1).sum()) == 2048
        buf = np.zeros(4096, dtype=np.uint8)
        us = timed(lambda: E.binding.lib().cmb200_residency(e.h, u, 0, (1 << 44) - 1, buf.ctypes.data), args.reps)
        assert int((buf == 1).sum()) == 2048
        print(json.dumps({"part": "residency", "table_slots": slots, "path": "scan", "pages": "whole object",
                          "us": round(us, 1)}), flush=True)
        e.close()


# ---- 2. usage ------------------------------------------------------------------------------------------------
def free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


if "2" not in skip:
    import torch
    torch.cuda.init()
    for n in (int(x) for x in args.usage_records.split(",")):
        for per in (int(x) for x in args.per_object.split(",")):
            slots = 1 << max(22, (2 * n - 1).bit_length())
            e = filled(slots, n, per, max(256 << 20, 96 * n))
            free0 = free_bytes()
            low = [free0]
            done = threading.Event()

            def poll():
                while not done.is_set():
                    low[0] = min(low[0], free_bytes())

            th = threading.Thread(target=poll)
            th.start()
            t = []
            for _ in range(args.usage_reps):
                t0 = time.perf_counter()
                cnt, rows = E.usage_set([e.h], 16)
                t.append(time.perf_counter() - t0)
            done.set()
            th.join()
            assert cnt == (n + per - 1) // per, (cnt, n, per)
            print(json.dumps({"part": "usage", "records": n, "pages_per_object": per, "objects": cnt,
                              "table_slots": slots, "ms_median": round(float(np.median(t)) * 1e3, 2),
                              "ms_min": round(min(t) * 1e3, 2), "runs": len(t),
                              "peak_scratch_mib": round((free0 - low[0]) / 2**20, 1),
                              "peak_scratch_bytes_per_record": round((free0 - low[0]) / n, 1)}), flush=True)
            e.close()


# ---- 3. serving while usage runs -------------------------------------------------------------------------------
if "3" not in skip:
    work = tempfile.mkdtemp(prefix="usage_serve_")
    exe = os.path.join(work, "usage_serve")
    libdir = os.path.dirname(E.library_path())
    subprocess.run(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tools", "usage_serve.c"), "-L" + libdir,
                    "-l:libcachemap.so.0.0", "-Wl,-rpath," + libdir, "-lpthread"], check=True)
    env = dict(os.environ, CMB200_PERSIST="0")
    for k in ("CMB200_DEVICES", "CMB200_HOST_TIER_MB", "CMB200_EVICT", "CMB200_ADMIT", "CMB200_GHOST"):
        env.pop(k, None)
    for threads in (8, 32):
        for with_usage in (0, 1):
            with tempfile.TemporaryDirectory(dir=work) as d:
                r = subprocess.run([exe, d, str(args.serve_pages), str(threads), str(args.serve_gets), str(with_usage)],
                                   capture_output=True, text=True, env=env, timeout=1200)
                assert r.returncode == 0, r.stdout + r.stderr
                print(json.dumps({"part": "serve", **json.loads(r.stdout.strip().splitlines()[-1])}), flush=True)
