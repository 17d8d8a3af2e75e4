"""Host tier measurements (DESIGN.md §2, §5, §12), all in one process tree on one GPU:

  1. demotion rate (cmb200_demote_batch), GiB/s of records, for incompressible (R) and text-like (T) pages;
  2. cmb200_get_small latency at 1..256 pages per call and cmb200_get_batch GiB/s, for the same pages in
     the HBM arena and in the host tier;
  3. drop-in cachemap_put_batch rate with a working set 4x the arena, host tier on and off (alternated);
  4. promotion rate (cmb200_promote_batch), GiB/s of records, 8 192 R or T records per call, and the
     cmb200_get_small latency of the same keys in the tier and after their promotion.

Every shape is warmed up first and every figure is repeated to show its spread.  The card's name and
power limit are recorded with the numbers.
usage: python tools/host_tier_bench.py [--only demotion,gets,drop_in,promotion] [--out FILE.json]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edge_fuse_b200 as E  # noqa: E402

BS = 65536
GIB = float(1 << 30)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def class_cids(cls, n):
    """The first n chunk ids of content class cls (streamgen.cuh: class = (cid + (cid >> 3)) & 3)."""
    return [c for c in range(8 * n) if ((c + (c >> 3)) & 3) == cls][:n]


def pages_of(kind, n, seed=11):
    return np.stack([E.gen_chunk_host(seed, c, BS) for c in class_cids({"R": 0, "T": 1}[kind], n)])


def demotion_rate(kind, reps=5):
    n = 8192                                                   # 512 MiB of pages per repetition
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 16, arena_bytes=4 << 30, max_batch=4096,
                   host_tier_bytes=8 << 30)
    pages = pages_of(kind, n)
    u = np.full(n, 1, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    rates = []
    for rep in range(reps + 1):                                # repetition 0 warms up
        eng.put(u, l, pages)                                   # fresh arena records for the same keys
        b0 = eng.host_tier_stats()["demoted_bytes"]
        t0 = time.perf_counter()
        moved = eng.demote(u, l)
        dt = time.perf_counter() - t0
        assert moved == n
        if rep:
            rates.append((eng.host_tier_stats()["demoted_bytes"] - b0) / dt / GIB)
        eng.compact()
    rec_kib = eng.host_tier_stats()["demoted_bytes"] / eng.host_tier_stats()["demoted_records"] / 1024
    eng.close()
    return {"kind": kind, "record_kib": round(rec_kib, 1), "gib_s": [round(r, 2) for r in rates]}


def gets(reps=5, iters=200):
    n = 4096
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 15, arena_bytes=2 << 30, max_batch=4096,
                   host_tier_bytes=2 << 30)
    pages = pages_of("T", n)
    l = np.arange(n, dtype=np.uint64)
    hbm, host = np.full(n, 2, dtype=np.uint64), np.full(n, 3, dtype=np.uint64)
    eng.put(hbm, l, pages)
    eng.put(host, l, pages)
    assert eng.demote(host, l) == n
    buf = E.lib().cmb200_host_alloc(256 * BS)
    status = np.zeros(256, dtype=np.int32)
    out = {"small_us": {}, "batch_gib_s": {}}
    for where, u in (("hbm", hbm), ("host", host)):
        for k in (1, 4, 16, 64, 256):
            times = []
            for it in range(iters + 20):                       # 20 warm-up calls of this shape
                at = (it * k) % (n - k)
                addr = np.ascontiguousarray(np.stack([u[at:at + k], l[at:at + k]], axis=1))
                t0 = time.perf_counter()
                rc = E.lib().cmb200_get_small(eng.h, k, addr.ctypes.data, buf, status.ctypes.data)
                dt = time.perf_counter() - t0
                assert rc == 0 and (status[:k] == E.HIT).all()
                if it >= 20:
                    times.append(dt * 1e6)
            p = np.percentile(times, [10, 50, 90])
            out["small_us"][f"{where}_{k}"] = [round(float(x), 1) for x in p]
        rates = []
        dst = np.zeros((n, BS), dtype=np.uint8)
        for rep in range(reps + 1):
            t0 = time.perf_counter()
            _, st = eng.get(u, l, out=dst)
            dt = time.perf_counter() - t0
            assert (st == E.HIT).all() and (dst == pages).all()
            if rep:
                rates.append(n * BS / dt / GIB)
        out["batch_gib_s"][where] = [round(r, 2) for r in rates]
    E.lib().cmb200_host_free(buf)
    out["host_tier_hits"] = eng.host_tier_stats()["hits"]
    eng.close()
    return out


DROP_IN = r'''
import os, sys, time, tempfile
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
pool = np.stack([E.gen_chunk_host(13, c, 65536) for c in range(4096) if ((c + (c >> 3)) & 3) == 1][:1024])   # text-like (T)
n, step = 32768, 4096                                     # 2 GiB of pages through a 512 MiB arena
with tempfile.TemporaryDirectory() as d:
    cm = E.Cachemap(d, 1 << 16, 12, 16)
    nh = np.full(step, 5, dtype=np.uint64); gen = np.zeros(step, dtype=np.uint32)
    pages = np.ascontiguousarray(pool[np.arange(step) % 1024])
    cm.put_batch(np.arange(step, dtype=np.uint64) << np.uint64(16), nh, gen, pages)   # warm-up (then overwritten)
    t0 = time.perf_counter()
    for base in range(0, n, step):
        cm.put_batch((np.arange(base, base + step, dtype=np.uint64) + np.uint64(1 << 20)) << np.uint64(16), nh, gen, pages)
    st = E.engine_stats(cm.engine_handle())                 # waits for the last batch
    dt = time.perf_counter() - t0
    ht = E.host_tier_stats(cm.engine_handle())
    print(n * 65536 / dt / 2**30, st["entries"], st["dropped_puts"], ht["demoted_records"])
    cm.free()
'''


def drop_in(reps=3):
    res = {"on": [], "off": []}
    for rep in range(reps):
        for mode in ("off", "on"):
            env = dict(os.environ, CMB200_ARENA_MB="512", CMB200_PERSIST="0")
            env.pop("CMB200_HOST_TIER_MB", None)
            if mode == "on":
                env["CMB200_HOST_TIER_MB"] = "4096"
            r = subprocess.run([sys.executable, "-c", DROP_IN], cwd=ROOT, env=env, capture_output=True, text=True,
                               timeout=1200)
            assert r.returncode == 0, r.stderr[-2000:]
            rate, entries, dropped, demoted = r.stdout.split()[-4:]
            res[mode].append({"gib_s": round(float(rate), 2), "entries": int(entries), "dropped_puts": int(dropped),
                              "demoted": int(demoted)})
    return res


def small_get_us(eng, u, l, k, buf, status, iters=200):
    """cmb200_get_small of k pages per call over the keys u, l: p10 / p50 / p90 microseconds."""
    n, times = len(u), []
    for it in range(iters + 20):                               # 20 warm-up calls of this shape
        at = (it * k) % (n - k)
        addr = np.ascontiguousarray(np.stack([u[at:at + k], l[at:at + k]], axis=1))
        t0 = time.perf_counter()
        rc = E.lib().cmb200_get_small(eng.h, k, addr.ctypes.data, buf, status.ctypes.data)
        dt = time.perf_counter() - t0
        assert rc == 0 and (status[:k] == E.HIT).all()
        if it >= 20:
            times.append(dt * 1e6)
    return [round(float(x), 1) for x in np.percentile(times, [10, 50, 90])]


def promotion(kind, reps=4):
    n = 8192                                                   # 512 MiB of pages per repetition
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 16, arena_bytes=4 << 30, max_batch=4096,
                   host_tier_bytes=4 << 30)
    pages = pages_of(kind, n)
    u = np.full(n, 1, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    eng.put(u, l, pages)
    rates = []
    for rep in range(reps + 1):                                # repetition 0 warms up
        assert eng.demote(u, l) == n
        eng.compact()                                          # the arena is empty: every record fits
        b0 = eng.host_tier_stats()["promoted_bytes"]
        t0 = time.perf_counter()
        moved = eng.promote(u, l)
        dt = time.perf_counter() - t0
        assert moved == n
        if rep:
            rates.append((eng.host_tier_stats()["promoted_bytes"] - b0) / dt / GIB)
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    # the same keys read from the tier, then after promotion
    buf = E.lib().cmb200_host_alloc(256 * BS)
    status = np.zeros(256, dtype=np.int32)
    lat = {}
    assert eng.demote(u, l) == n
    eng.compact()
    for k in (1, 64, 256):
        lat[f"tier_{k}"] = small_get_us(eng, u, l, k, buf, status)
    assert eng.promote(u, l) == n
    for k in (1, 64, 256):
        lat[f"promoted_{k}"] = small_get_us(eng, u, l, k, buf, status)
    E.lib().cmb200_host_free(buf)
    rec_kib = eng.host_tier_stats()["promoted_bytes"] / eng.host_tier_stats()["promoted_records"] / 1024
    eng.close()
    return {"kind": kind, "record_kib": round(rec_kib, 1), "gib_s": [round(r, 2) for r in rates], "small_us": lat}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="demotion,gets,drop_in,promotion", help="sections to run")
    ap.add_argument("--out", help="also write the result here")
    a = ap.parse_args()
    only = set(a.only.split(","))
    assert E.device_count() > 0, f"no CUDA device: {E.last_error()}"
    res = {"card": card()}
    if "demotion" in only:
        res["demotion"] = [demotion_rate("R"), demotion_rate("T")]
        print(json.dumps(res), flush=True)
    if "gets" in only:
        res["gets"] = gets()
        print(json.dumps(res["gets"]), flush=True)
    if "promotion" in only:
        res["promotion"] = [promotion("R"), promotion("T")]
        print(json.dumps(res["promotion"]), flush=True)
    if "drop_in" in only:
        res["drop_in_put_4x_arena"] = drop_in()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
