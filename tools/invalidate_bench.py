"""Cost of cmb200_invalidate and cachemap_invalidate, and the interval length at which the engine's
page-by-page path (k_invalidate_keys) and its table scan (k_invalidate_scan) cost the same.

- scan: an interval longer than any table, on tables of 2^20, 2^23, 2^25 and 2^27 slots with a small
  arena.  The scan reads 32 B of every one of the cap + 2 slots; the achieved rate of those bytes is
  put against the H100 SXM data sheet's 3.35 TB/s.
- keyed: 1, 16, 256, 4096 and 65536 cached pages of one object removed per call, on 2^25 and 2^27
  tables.  The pages are put again (untimed) before every call.  The crossover is where the line
  through the two longest keyed counts meets the scan's time on the same table.
- drop-in: a rename at 4 KiB pages (cachemap_invalidate of both names, CACHEMAP_TO_END), with the
  write-behind ring idle and with 8 threads putting pages (the drain of the ring is part of the call).

Times are per call: a host clock around the call, which ends in a synchronise of the engine's stream.
Median and p10-p90 of --reps calls after --warmup.  The card's name and power limit are read in the
same run.  One JSON line per measurement.

usage: python tools/invalidate_bench.py [--reps 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import edge_fuse_b200 as E  # noqa: E402

TO_END = (1 << 64) - 1
HBM_DATASHEET = 3.35e12          # H100 SXM, bytes/s


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def summary(ts):
    us = np.array(ts) * 1e6
    return {"median_us": round(float(np.median(us)), 2), "p10_us": round(float(np.percentile(us, 10)), 2),
            "p90_us": round(float(np.percentile(us, 90)), 2), "calls": len(us)}


def timed(fn, reps, warmup, before=None):
    out = []
    for i in range(warmup + reps):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        if i >= warmup:
            out.append(t1 - t0)
    return out


def engine(slots):
    return E.Engine(pshift=12, accel=12, capacity=1 << 16, table_slots=slots, arena_bytes=1 << 30, max_batch=4096)


def fill(eng, u, n, zeros):
    """puts pages 0..n of object u (untimed)."""
    for at in range(0, n, 4096):
        m = min(4096, n - at)
        eng.put(np.full(m, u, dtype=np.uint64), np.arange(at, at + m, dtype=np.uint64), zeros[:m])


def scan_bench(slots, reps, warmup, gpu):
    eng = engine(slots)
    cap = eng.stats()["table_slots"]
    ts = timed(lambda: eng.invalidate(99, 0, TO_END), reps, warmup)
    s = summary(ts)
    gbs = 32 * (cap + 2) / (s["median_us"] * 1e-6) / 1e9
    res = {"bench": "scan", "gpu": gpu, "table_slots": cap, "bytes_per_call": 32 * (cap + 2), **s,
           "achieved_GBps": round(gbs, 1), "of_datasheet_3350GBps": round(gbs * 1e9 / HBM_DATASHEET, 3)}
    eng.close()
    return res


def keyed_bench(slots, counts, reps, warmup, gpu, zeros):
    eng = engine(slots)
    cap = eng.stats()["table_slots"]
    scan = summary(timed(lambda: eng.invalidate(99, 0, TO_END), reps, warmup))
    rows = []
    for n in counts:
        assert n - 1 < (cap + 2) // 64, "a keyed count must stay below the scan threshold"
        removed = []
        ts = timed(lambda: removed.append(eng.invalidate(7, 0, n - 1)), reps, warmup, before=lambda: fill(eng, 7, n, zeros))
        assert all(r == n for r in removed), (n, set(removed))
        rows.append({"pages": n, **summary(ts)})
    (n1, t1), (n2, t2) = [(r["pages"], r["median_us"]) for r in rows[-2:]]
    slope = (t2 - t1) / (n2 - n1)
    cross = (scan["median_us"] - (t1 - slope * n1)) / slope if slope > 0 else float("inf")
    res = {"bench": "keyed", "gpu": gpu, "table_slots": cap, "scan": scan, "keyed": rows,
           "crossover_pages": round(cross), "crossover_over_slots": round(cross / (cap + 2), 4)}
    eng.close()
    return res


def drop_in_bench(reps, warmup, gpu, busy):
    os.environ["CMB200_PERSIST"] = "0"
    d = tempfile.mkdtemp()
    cm = E.Cachemap(d, 1 << 18, 12, 12)
    page = np.frombuffer(np.random.default_rng(1).integers(0, 16, 4096, dtype=np.uint8).tobytes(), dtype=np.uint8)

    def cache_both():
        for nh in (50, 51):
            for i in range(64):
                cm.put(i << 12, nh, 0, page)

    stop = threading.Event()

    def putter(k):
        i = 0
        while not stop.is_set():
            cm.put((i % 16384) << 12, 1000 + k, 0, page)
            i += 1

    th = [threading.Thread(target=putter, args=(k,)) for k in range(8 if busy else 0)]
    for t in th:
        t.start()
    ts = timed(lambda: (cm.invalidate(50, 0, 0, cm.TO_END), cm.invalidate(51, 0, 0, cm.TO_END)), reps, warmup,
               before=cache_both)
    stop.set()
    for t in th:
        t.join()
    cm.free()
    return {"bench": "drop_in_rename", "gpu": gpu, "page": 4096, "ring": "busy, 8 putting threads" if busy else "idle",
            **summary(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    gpu = card()
    zeros = np.zeros((4096, 4096), dtype=np.uint8)
    for p in (20, 23, 25, 27):
        print(json.dumps(scan_bench(1 << p, a.reps, a.warmup, gpu)), flush=True)
    for p in (25, 27):
        print(json.dumps(keyed_bench(1 << p, [1, 16, 256, 4096, 65536], a.reps, a.warmup, gpu, zeros)), flush=True)
    for busy in (False, True):
        print(json.dumps(drop_in_bench(a.reps, a.warmup, gpu, busy)), flush=True)


if __name__ == "__main__":
    main()
