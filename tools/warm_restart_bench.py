"""Restart of a saved store through the drop-in, loading before serving (CMB200_LOAD=wait) against loading
in the background (CMB200_LOAD=background).

For each page size a store of --gib GiB of page data is put through cachemap_put_batch and saved by
cachemap_free.  Then the map is restarted --rounds times in each mode, the modes alternated.  Reported per
restart: the time from cachemap_create to the first answered cachemap_get; cachemap_get p50 / p99 / max
latency from 8 threads while the load runs (for "wait", over the same window after the first answer);
the rate of cachemap_put from one more thread meanwhile; and the total load time (until
cachemap_load_progress reports the load done).  Each restart loads the file fill saved.  The card's
name and power limit are read in the same run.  One JSON line per page size.

usage: python tools/warm_restart_bench.py [--gib 4] [--pshift 12 16] [--rounds 2] [--dir /tmp]
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

NH = 7
READERS = 8


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def fill(d, pshift, n):
    bs = 1 << pshift
    rng = np.random.default_rng(pshift)
    # half the bytes from a 16-letter alphabet: LZ4 keeps about 60 % of such a page
    chunk = min(n, (256 << 20) // bs)
    pg = rng.integers(0, 16, size=(chunk, bs), dtype=np.uint8)
    pg[:, bs // 2:] = 0x41
    cm = E.Cachemap(d, int(n * 1.25), 12, pshift)
    for at in range(0, n, chunk):
        m = min(chunk, n - at)
        off = (np.arange(at, at + m, dtype=np.uint64) << np.uint64(pshift))
        cm.put_batch(off, np.full(m, NH, dtype=np.uint64), np.ones(m, dtype=np.uint32), pg[:m])
    cm.free()


def restart(d, pshift, n, mode):
    bs = 1 << pshift
    os.environ["CMB200_LOAD"] = mode
    t0 = time.perf_counter()
    cm = E.Cachemap(d, int(n * 1.25), 12, pshift)
    cm.get(0, NH, 1)
    first = time.perf_counter() - t0
    stop = threading.Event()
    lat = [[] for _ in range(READERS)]
    hits = [0] * READERS
    puts = [0]

    def reader(k):
        r = np.random.default_rng(100 + k)
        while not stop.is_set():
            p = int(r.integers(0, n))
            s = time.perf_counter()
            got = cm.get(p << pshift, NH, 1)
            lat[k].append(time.perf_counter() - s)
            hits[k] += got is not None

    def putter():
        page = np.full(bs, 0x42, dtype=np.uint8)
        i = 0
        while not stop.is_set():
            cm.put((n + (i % 65536)) << pshift, NH, 1, page)
            i += 1
        puts[0] = i

    threads = [threading.Thread(target=reader, args=(k,)) for k in range(READERS)] + [threading.Thread(target=putter)]
    for th in threads:
        th.start()
    t1 = time.perf_counter()
    while cm.load_progress()[0]:
        time.sleep(0.005)
    loaded = time.perf_counter() - t0
    if mode == "wait":
        time.sleep(1.0)                 # a window of serving after the load, for the same figures
    window = time.perf_counter() - t1
    stop.set()
    for th in threads:
        th.join()
    ms = np.concatenate([np.array(x) for x in lat]) * 1e3 if any(lat) else np.zeros(1)
    out = dict(mode=mode, first_get_s=round(first, 4), load_s=round(loaded, 3), window_s=round(window, 3),
               gets=int(ms.size), get_hit_frac=round(sum(hits) / max(ms.size, 1), 4),
               get_ms_p50=round(float(np.percentile(ms, 50)), 4), get_ms_p99=round(float(np.percentile(ms, 99)), 4),
               get_ms_max=round(float(ms.max()), 3), puts_per_s=round(puts[0] / window, 1))
    cm.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4)
    ap.add_argument("--pshift", type=int, nargs="*", default=[12, 16])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    a = ap.parse_args()
    for k in ("CMB200_DEVICES", "CMB200_HOST_TIER_MB", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        os.environ.pop(k, None)
    for pshift in a.pshift:
        n = int(a.gib * (1 << 30)) >> pshift
        d = tempfile.mkdtemp(dir=a.dir)
        fill(d, pshift, n)
        snap = os.path.join(d, "cachemap_b200.snap")
        saved = snap + ".saved"
        shutil.copyfile(snap, saved)
        res = dict(pshift=pshift, pages=n, file_bytes=os.path.getsize(snap), card=card(), restarts=[])
        for _ in range(a.rounds):
            for mode in ("wait", "background"):
                # every restart loads the same file: cachemap_free saves the pages the putter added
                shutil.copyfile(saved, snap)
                res["restarts"].append(restart(d, pshift, n, mode))
        shutil.rmtree(d)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
