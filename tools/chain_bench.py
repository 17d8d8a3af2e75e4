"""Cost of snapshot-chain ticks (cmb200_chain_begin) against full saves of the same store.

For each page size (64 KiB and 4 KiB pages) a store of --gib GiB of page data is put into one engine,
then a base is written, and for each churn level (0 %, 1 %, 10 %, 50 % of the keys rewritten, plus 0.1 %
unset) one delta tick follows.  Reported per tick: file bytes and wall time against a full save
(cmb200_save) of the same store; how long the tick held the engine (cmb200_chain_begin: export +
k_delta_gone under the lock); p50 / p99 / max of back-to-back 64-page put batches while the tick runs;
and the load time of base + deltas (cmb200_load_chain) against one full file.  One JSON line per page
size; the card's name and power limit are read in the same run.

usage: python tools/chain_bench.py [--gib 8] [--dir /tmp]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import edge_fuse_b200 as E  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def pages(rng, n, bs):
    # half the bytes from a 16-letter alphabet: LZ4 keeps about 60 % of such a page
    p = rng.integers(0, 16, size=(n, bs), dtype=np.uint8)
    p[:, bs // 2:] = 0x41
    return p


def put_keys(eng, keys, bs, rng, batch):
    for at in range(0, len(keys), batch):
        k = keys[at:at + batch]
        eng.put(np.full(len(k), 7, dtype=np.uint64), k.astype(np.uint64), pages(rng, len(k), bs))


def timed_tick(eng, base, delta, bs, rng):
    """-> (seconds held in begin, seconds to finish, put latencies during the tick)."""
    lat, stop = [], threading.Event()
    keys = np.arange(1 << 40, (1 << 40) + 64, dtype=np.uint64)

    def putter():
        while not stop.is_set():
            t0 = time.perf_counter()
            eng.put(np.full(64, 9, dtype=np.uint64), keys, pages(rng, 64, bs))
            lat.append(time.perf_counter() - t0)

    th = threading.Thread(target=putter)
    th.start()
    time.sleep(0.05)
    t0 = time.perf_counter()
    s = E.chain_begin([eng.h], base, delta)
    t1 = time.perf_counter()
    E.snapshot_finish(s)
    t2 = time.perf_counter()
    stop.set()
    th.join()
    return t1 - t0, t2 - t0, lat


def run(pshift, gib, tmp):
    bs = 1 << pshift
    n = (gib << 30) // bs
    rng = np.random.default_rng(pshift)
    eng = E.Engine(pshift=pshift, accel=12, capacity=int(n * 1.3), arena_bytes=int(gib * 1.6) << 30,
                   max_batch=4096)
    keys = np.arange(n, dtype=np.uint64)
    put_keys(eng, keys, bs, rng, 4096)
    d = tempfile.mkdtemp(dir=tmp)
    full = os.path.join(d, "full.snap")
    t0 = time.perf_counter()
    eng.save(full)
    full_s = time.perf_counter() - t0
    full_bytes = os.path.getsize(full)
    base = os.path.join(d, "chain.snap")
    hold, wall, _ = timed_tick(eng, base, False, bs, rng)
    out = dict(pshift=pshift, pages=int(n), store_gib=gib, card=card(), full_save_s=round(full_s, 3),
               full_bytes=full_bytes, base=dict(s=round(wall, 3), locked_s=round(hold, 4)), ticks=[])
    for churn in (0.0, 0.01, 0.10, 0.50):
        m = int(n * churn)
        put_keys(eng, rng.choice(keys, m, replace=False), bs, rng, 4096)
        gone = rng.choice(keys, n // 1000, replace=False)
        eng.unset(np.full(len(gone), 7, dtype=np.uint64), gone)
        hold, wall, lat = timed_tick(eng, base, True, bs, rng)
        k = len(out["ticks"]) + 1
        lat_ms = np.array(lat) * 1e3 if lat else np.zeros(1)
        out["ticks"].append(dict(churn=churn, rewritten=m, unset=len(gone), bytes=os.path.getsize(f"{base}.d{k}"),
                                 s=round(wall, 3), locked_s=round(hold, 4), vs_full_bytes=round(os.path.getsize(f"{base}.d{k}") / full_bytes, 4),
                                 vs_full_time=round(wall / full_s, 4), put_ms_p50=round(float(np.percentile(lat_ms, 50)), 3),
                                 put_ms_p99=round(float(np.percentile(lat_ms, 99)), 3), put_ms_max=round(float(lat_ms.max()), 3),
                                 put_batches=len(lat)))
    geo = dict(pshift=pshift, accel=12, capacity=int(n * 1.3), arena_bytes=int(gib * 1.6) << 30, max_batch=4096)
    eng.save(full)
    eng.close()
    for name, fn in (("load_full_s", lambda e: e.load(full)), ("load_chain_s", lambda e: E.load_chain([e.h], base))):
        e = E.Engine(**geo)
        t0 = time.perf_counter()
        fn(e)
        out[name] = round(time.perf_counter() - t0, 3)
        e.close()
    shutil.rmtree(d)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=int, default=8)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--pshift", type=int, nargs="*", default=[16, 12])
    a = ap.parse_args()
    for p in a.pshift:
        print(json.dumps(run(p, a.gib, a.dir)), flush=True)


if __name__ == "__main__":
    main()
