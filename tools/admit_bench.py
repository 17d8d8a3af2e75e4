#!/usr/bin/env python
"""What CMB200_ADMIT=freq costs and buys.

1. Hit ratios: the hot and cold workload and the scan workload of tests/admit_model.py through the drop-in
   (cachemap_get, cachemap_put on a miss) at --capacity pages of 4 KiB, synchronous puts, under
   CMB200_EVICT=put, =access, and =access with CMB200_ADMIT=freq, next to the model's values for the same
   workload, drawing as the store does (model_table).
   Each run also reports its synchronous cachemap_put time after the warm-up (median and p90 microseconds,
   host clock): at capacity every put evicts, and with CMB200_ADMIT=freq it asks the sketch for estimates.
2. Latency of cmb200_get_small (host clock around calls that return when the pages are in page-locked
   memory, median and p10-p90 microseconds) on an engine without the flag and one with CMB200_FREQ holding
   the same records, alternated call by call, at 1 and 132 pages per call and 64 KiB pages.
3. Throughput of concurrent cmb200_get_small calls of one page each from --threads host threads on one
   engine (calls per second, median of three rounds that alternate the engine without and with the flag).
The card's name and power limit are printed first: they belong beside the numbers."""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import admit_model as A
import edge_fuse_b200 as E

ap = argparse.ArgumentParser()
ap.add_argument("--capacity", type=int, default=65536, help="pages of the drop-in map")
ap.add_argument("--steps", type=int, default=131072)
ap.add_argument("--warmup", type=int, default=65536)
ap.add_argument("--sizes", default="1,132", help="pages per cmb200_get_small call")
ap.add_argument("--reps", type=int, default=200)
ap.add_argument("--skip-ratios", action="store_true")
ap.add_argument("--threads", default="1,8,32", help="host threads of the concurrent get_small measurement")
ap.add_argument("--thread-calls", type=int, default=2000, help="calls per thread per round")
args = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip()
except OSError:
    card = "unknown"
print(json.dumps({"card": card}), flush=True)
assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"

POLICIES = {"put": ("put", "all"), "access": ("access", "all"), "access+freq": ("access", "freq")}
WORKLOADS = {"hot_cold": args.capacity // 4, "scan": args.capacity // 2}      # hot-set size


def dropin_ratio(workload: str, evict: str, admit: str, d: str, seed: int = 1):
    """-> (hot-set hit ratio after the warm-up, (admitted, rejected), seconds) through the drop-in."""
    os.environ.update(CMB200_EVICT=evict, CMB200_ADMIT=admit, CMB200_PERSIST="0", CMB200_WB_SLOTS="0")
    E.binding._libc().srand(seed)
    cm = E.Cachemap(d, args.capacity, 12, 12)
    hot = WORKLOADS[workload]
    rng = random.Random(seed ^ 0x5CA7)
    page = np.zeros(4096, dtype=np.uint8)
    hits = reads = 0
    put_us = []

    def put(off, nhid):
        t1 = time.perf_counter()
        cm.put(off, nhid, 0, page)
        if t >= args.warmup:
            put_us.append((time.perf_counter() - t1) * 1e6)

    t0 = time.perf_counter()
    for t in range(args.steps):
        h = t % hot if workload == "hot_cold" else rng.randrange(hot)
        hit = cm.get(h << 12, A.HOT_NHID, 0) is not None
        if not hit:
            put(h << 12, A.HOT_NHID)
        if workload == "scan":
            cm.get(t << 12, A.COLD_NHID, 0)           # read once, a miss: the scan page is put
        put(t << 12, A.COLD_NHID)
        if t >= args.warmup:
            reads += 1
            hits += hit
    adm = cm.admission()
    cm.free()
    return hits / reads, adm, time.perf_counter() - t0, [round(float(x), 1) for x in np.percentile(put_us, [50, 90])]


def model_ratio(workload: str, evict: str, admit: str, seed: int = 1) -> float:
    fn = A.hot_cold if workload == "hot_cold" else A.scan
    return fn(evict == "access", admit == "freq", args.capacity, WORKLOADS[workload], steps=args.steps,
              warmup=args.warmup, seed=seed, table=True)


if not args.skip_ratios:
    for workload in WORKLOADS:
        row = {}
        for name, (evict, admit) in POLICIES.items():
            with tempfile.TemporaryDirectory() as d:
                r, adm, s, put_us = dropin_ratio(workload, evict, admit, d)
            row[name] = {"dropin": round(r, 4), "model_table": round(model_ratio(workload, evict, admit), 4),
                         "admitted": adm[0], "rejected": adm[1], "seconds": round(s, 1), "put_us_p50_p90": put_us}
        print("hit_ratio", workload, json.dumps({"capacity": args.capacity, "hot": WORKLOADS[workload],
                                                 "steps": args.steps, "warmup": args.warmup, **row}), flush=True)

# ---- cmb200_get_small latency, flag off and on --------------------------------------------------
PSHIFT = 16
CH = 1 << PSHIFT
sizes = [int(s) for s in args.sizes.split(",")]
n = max(sizes)
GEO = dict(pshift=PSHIFT, accel=12, capacity=1 << 16, arena_bytes=2 << 30, max_batch=1024)
engines = {"off": E.Engine(**GEO), "freq": E.Engine(**GEO, flags=E.FREQ)}
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
            for _ in range(args.reps):                # off and freq alternate call by call
                for name, fn in calls:
                    t0 = time.perf_counter()
                    fn()
                    t[name].append((time.perf_counter() - t0) * 1e6)
            for name, v in t.items():
                p10, p50, p90 = np.percentile(v, [10, 50, 90])
                row[name] = [round(p50, 1), round(p10, 1), round(p90, 1)]
        print("get_small", cls, json.dumps(row), flush=True)
    print("freq_stats", json.dumps(engines["freq"].freq_stats()), flush=True)

    # ---- concurrent single-page gets: T threads on one engine, each with its own page-locked page ----
    L = E.lib()

    def rate(eng, threads):
        bufs = [L.cmb200_host_alloc(CH) for _ in range(threads)]
        addrs = [np.array([[u[0], l[k % n]]], dtype=np.uint64) for k in range(threads)]
        stats = [np.zeros(1, dtype=np.int32) for _ in range(threads)]
        go = threading.Barrier(threads + 1)

        def work(k):
            a, st, b = addrs[k].ctypes.data, stats[k].ctypes.data, bufs[k]
            go.wait()
            for _ in range(args.thread_calls):
                L.cmb200_get_small(eng.h, 1, a, b, st)

        ths = [threading.Thread(target=work, args=(k,)) for k in range(threads)]
        for th in ths:
            th.start()
        go.wait()
        t0 = time.perf_counter()
        for th in ths:
            th.join()
        dt = time.perf_counter() - t0
        assert all(st[0] == E.HIT for st in stats)
        for b in bufs:
            L.cmb200_host_free(b)
        return threads * args.thread_calls / dt

    for threads in [int(x) for x in args.threads.split(",")]:
        got = {w: [] for w in engines}
        for _ in range(3):                            # off and freq alternate round by round
            for w, eng in engines.items():
                got[w].append(rate(eng, threads))
        print("get_small_threads", json.dumps({"threads": threads, "pages_per_call": 1, "content": "M",
                                               **{f"{w}_calls_per_s": round(float(np.median(v))) for w, v in got.items()}}),
              flush=True)
finally:
    E.lib().cmb200_host_free(hp)
    for eng in engines.values():
        eng.close()
