"""Ghost entries (CMB200_GHOST): how well the hit curve predicts a larger store, and what the probes cost.

Accuracy, through the drop-in at 4 KiB pages with synchronous puts (every get and put reaches the GPU): each
workload of tests/ghost_model.py (hot/cold, a hot set with a scan, zipf 0.9) under CMB200_EVICT=put and
=access runs once at capacity C with CMB200_GHOST=1, which gives the measured hit ratio and the predicted
ones at 1.5 C and 2 C (cachemap_hit_curve's refaults of the measured gets added to its hits), then without the
flag at 1.5 C and 2 C for the real ones.

Cost: cmb200_get_small of one page (half hits, half misses that probe) from 1, 8 and 32 threads, on an engine
without and one with the flag, alternated over rounds: the median and p10-p90 latency of a call and calls per
second; and how often cmb200_get_small_begin found a lane's previous probe still running, and for how long.

The card's name and power limit are read in the same run.  Prints one JSON object.
    python tools/ghost_bench.py [--capacity 4096] [--rounds 4] [--skip-accuracy] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import edge_fuse_b200 as E  # noqa: E402
import ghost_model as G  # noqa: E402

WORKLOADS = {"hot_cold": dict(hot=2048), "scan": dict(hot=4096), "zipf": dict(keys=40000)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def dropin_run(workload, evict, capacity, ghost, steps, warmup, seed, extra=()):
    env = {"CMB200_PERSIST": "0", "CMB200_WB_SLOTS": "0", "CMB200_EVICT": evict}
    for k in ("CMB200_DEVICES", "CMB200_ADMIT", "CMB200_HOST_TIER_MB", "CMB200_GHOST"):
        os.environ.pop(k, None)
    os.environ.update(env)
    if ghost:
        os.environ["CMB200_GHOST"] = "1"
    E.binding._libc().srand(seed)
    with tempfile.TemporaryDirectory() as d:
        cm = E.Cachemap(d, capacity, 12, 12)
        page = np.zeros(1 << 12, dtype=np.uint8)
        hits = reads = 0
        curve0 = None
        kw = WORKLOADS[workload]
        per_step = 2 if workload in ("hot_cold", "scan") else 1
        try:
            for t, (a, read) in enumerate(G._reads(workload, steps, seed, kw.get("hot", 0), kw.get("keys", 0), 0.9)):
                measured = t >= warmup * per_step
                if ghost and t == warmup * per_step:
                    curve0, _ = cm.hit_curve(list(extra))
                if read:
                    hit = cm.get(a[1] << 12, a[0], 0) is not None
                    if measured:
                        reads += 1
                        hits += hit
                    if hit:
                        continue
                page[:8] = np.frombuffer(np.uint64(a[1]).tobytes(), dtype=np.uint8)
                cm.put(a[1] << 12, a[0], 0, page)
            pred = {}
            if ghost:
                curve, _ = cm.hit_curve(list(extra))
                pred = {x: (hits + int(c) - int(c0)) / reads for x, c, c0 in zip(extra, curve, curve0)}
        finally:
            cm.free()
            os.environ.pop("CMB200_GHOST", None)
    return hits / reads, pred


def accuracy(capacity, steps, warmup):
    out = []
    extra = (capacity // 2, capacity)
    for workload in WORKLOADS:
        for evict in ("put", "access"):
            base, pred = dropin_run(workload, evict, capacity, True, steps, warmup, 1, extra)
            row = {"workload": workload, "evict": evict, "capacity": capacity, "hit_ratio": round(base, 4)}
            for x, name in zip(extra, ("1.5x", "2x")):
                real, _ = dropin_run(workload, evict, capacity + x, False, steps, warmup, 1)
                row[name] = {"predicted": round(pred[x], 4), "real": round(real, 4), "error": round(pred[x] - real, 4)}
            out.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    return out


def small_get_cost(rounds, calls_per_thread):
    n, bs = 4096, 1 << 12
    engines = {}
    for name, flags in (("off", 0), ("on", E.GHOST)):
        e = E.Engine(pshift=12, capacity=n, arena_bytes=256 << 20, max_batch=1024, flags=flags)
        u = np.full(n, 9, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        e.put(u, l, np.random.default_rng(1).integers(0, 256, size=(n, bs), dtype=np.uint8))
        if flags:
            e.evict(u[n // 2:], l[n // 2:])        # the misses below find ghosts until they are consumed
        else:
            e.unset(u[n // 2:], l[n // 2:])
        engines[name] = e
    res = {name: {t: [] for t in (1, 8, 32)} for name in engines}
    rate = {name: {t: [] for t in (1, 8, 32)} for name in engines}

    def worker(e, lat, seed):
        rng = np.random.default_rng(seed)
        out = E.lib().cmb200_host_alloc(bs)
        addr = np.zeros((1, 2), dtype=np.uint64)
        st = np.zeros(1, dtype=np.int32)
        try:
            for _ in range(calls_per_thread):
                addr[0] = (9, int(rng.integers(0, n)))
                t0 = time.perf_counter_ns()
                E.lib().cmb200_get_small(e.h, 1, addr.ctypes.data, out, st.ctypes.data)
                lat.append(time.perf_counter_ns() - t0)
        finally:
            E.lib().cmb200_host_free(out)

    for r in range(rounds):
        for threads in (1, 8, 32):
            for name in (("off", "on") if r % 2 == 0 else ("on", "off")):
                lats = [[] for _ in range(threads)]
                ths = [threading.Thread(target=worker, args=(engines[name], lats[k], 1000 * r + k)) for k in range(threads)]
                t0 = time.perf_counter()
                for th in ths:
                    th.start()
                for th in ths:
                    th.join()
                wall = time.perf_counter() - t0
                res[name][threads].extend(x for lat in lats for x in lat)
                rate[name][threads].append(threads * calls_per_thread / wall)
    summary = {}
    for name in engines:
        summary[name] = {}
        for threads, lat in res[name].items():
            a = np.array(lat) / 1000.0
            summary[name][threads] = {"median_us": round(float(np.median(a)), 2),
                                      "p10_us": round(float(np.percentile(a, 10)), 2),
                                      "p90_us": round(float(np.percentile(a, 90)), 2),
                                      "calls_per_s": round(float(np.median(rate[name][threads])), 0)}
    st = engines["on"].ghost_stats()
    summary["lane_waits"] = st["lane_waits"]
    summary["lane_wait_us"] = round(st["lane_wait_ns"] / 1000.0, 1)
    summary["probes"] = st["probes"]
    summary["small_gets"] = int(sum(len(v) for v in res["on"].values()))
    for e in engines.values():
        e.close()
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=48000)
    ap.add_argument("--warmup", type=int, default=16000)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--calls", type=int, default=2000, help="small gets per thread per round")
    ap.add_argument("--skip-accuracy", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"
    result = {"card": card()}
    if not args.skip_accuracy:
        result["accuracy"] = accuracy(args.capacity, args.steps, args.warmup)
    result["get_small"] = small_get_cost(args.rounds, args.calls)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
