"""Cost of CMB200_VERIFY on the GPU: the same gets on two engines, one created without the flag and one
with it, taken in alternation so that both see the same machine state.

  * cmb200_get_small: median and p10-p90 microseconds per call at 1 / 32 / 132 pages, T and R pages,
    pshift 16 and 17;
  * cmb200_get_batch_dev: GiB/s over 4096 pages (pshift 16, T);
  * cmb200_verify_store: records/s and GiB/s of pages, the records in HBM and in the host tier.

Prints one JSON object, with the card's name and power limit read in the same run (and writes it to
--out when given).
Usage: python tools/verify_bench.py [--reps 200] [--out result.json]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import edge_fuse_b200 as E  # noqa: E402
import datagen  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().splitlines() or ["?,?,?"])[0].split(", ")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def engines(pshift, tier=0, count=4096):
    return [E.Engine(pshift=pshift, capacity=count, arena_bytes=(count + 64) << (pshift + 1), flags=f,
                     host_tier_bytes=tier) for f in (0, E.VERIFY)]


def keys(n):
    return np.full(n, 5, dtype=np.uint64), np.arange(n, dtype=np.uint64)


def small_gets(reps):
    out = {}
    for pshift in (16, 17):
        n = 1 << pshift
        for kind in ("T", "R"):
            pages = np.stack([datagen.make_page(kind, n, 50 + i) for i in range(132)])
            u, l = keys(132)
            es = engines(pshift, count=256)
            for e in es:
                e.put(u, l, pages)
            buf = E.lib().cmb200_host_alloc(132 * n)
            try:
                for m in (1, 32, 132):
                    addr = np.stack([u[:m], l[:m]], axis=1).astype(np.uint64)
                    st = np.zeros(m, dtype=np.int32)
                    t = {0: [], 1: []}
                    for r in range(reps + 10):
                        for k, e in enumerate(es):
                            t0 = time.perf_counter()
                            rc = E.lib().cmb200_get_small(e.h, m, addr.ctypes.data, buf, st.ctypes.data)
                            dt = time.perf_counter() - t0
                            assert rc == 0 and (st == E.HIT).all()
                            if r >= 10:
                                t[k].append(dt * 1e6)
                    for k, name in ((0, "off"), (1, "verify")):
                        a = np.array(t[k])
                        out[f"get_small p{pshift} {kind} x{m} {name}"] = {
                            "median_us": round(float(np.median(a)), 1),
                            "p10_us": round(float(np.percentile(a, 10)), 1),
                            "p90_us": round(float(np.percentile(a, 90)), 1)}
                assert es[1].verify_stats()["corrupt"] == 0
            finally:
                E.lib().cmb200_host_free(buf)
                for e in es:
                    e.close()
    return out


def batch_dev(reps):
    pshift, count = 16, 4096
    n = 1 << pshift
    pages = np.stack([datagen.make_page("T", n, 900 + i) for i in range(count)])
    u, l = keys(count)
    es = engines(pshift, count=count)
    addr = np.stack([u, l], axis=1).astype(np.uint64)
    st = np.zeros(count, dtype=np.int32)
    out = {}
    t = {0: [], 1: []}
    devs = [E.lib().cmb200_dev_alloc(e.h, count * n) for e in es]
    try:
        for e in es:
            e.put(u, l, pages)
        for r in range(reps + 2):
            for k, e in enumerate(es):
                t0 = time.perf_counter()
                rc = E.lib().cmb200_get_batch_dev(e.h, count, addr.ctypes.data, None, devs[k], st.ctypes.data)
                dt = time.perf_counter() - t0
                assert rc == 0 and (st == E.HIT).all()
                if r >= 2:
                    t[k].append(dt)
        for k, name in ((0, "off"), (1, "verify")):
            out[f"get_batch_dev p16 T x4096 {name} GiB/s"] = round(count * n / float(np.median(t[k])) / 2**30, 2)
    finally:
        for e, d in zip(es, devs):
            E.lib().cmb200_dev_free(e.h, d)
            e.close()
    return out


def store_scan():
    pshift, count = 16, 4096
    n = 1 << pshift
    pages = np.stack([datagen.make_page("TRZM"[i % 4], n, 300 + i) for i in range(count)])
    u, l = keys(count)
    e = E.Engine(pshift=pshift, capacity=count, arena_bytes=(count + 64) << (pshift + 1), flags=E.VERIFY,
                 host_tier_bytes=(count + 64) << (pshift + 1))
    out = {}
    try:
        e.put(u, l, pages)
        for where in ("hbm", "tier"):
            if where == "tier":
                assert e.demote(u, l) == count
            e.verify_store()
            t0 = time.perf_counter()
            _, _, bad, checked = e.verify_store()
            dt = time.perf_counter() - t0
            assert bad == 0 and checked == count
            out[f"verify_store {where} records/s"] = round(count / dt)
            out[f"verify_store {where} page GiB/s"] = round(count * n / dt / 2**30, 2)
    finally:
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert E.device_count() > 0, E.last_error()
    res = card()
    res.update(small_gets(args.reps))
    res.update(batch_dev(max(5, args.reps // 20)))
    res.update(store_scan())
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
