#!/usr/bin/env python
"""One map over 1, 2, ..., N engines (CMB200_DEVICES = the first k devices; on a one-GPU machine "0" and
"0,0", which measures the cost of the routing alone).  For each list, from native threads:
cachemap_get GiB/s at 8 and 32 callers (tools/api_threads.c, one 64 KiB page per call; its cachemap_put
rate is reported too), and cachemap_put_batch / cachemap_get_batch GiB/s (batches of 4096 64 KiB pages
in host memory from one caller).
Prints the card name and power limit read in the same run, and one JSON object on the last line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import edge_fuse_b200 as E

PUT_BATCH = r'''
import os, sys, time, tempfile
sys.path.insert(0, sys.argv[1])
import numpy as np, edge_fuse_b200 as E
pages = np.fromfile(sys.argv[2], dtype=np.uint8).reshape(-1, 65536)
n, reps = 4096, int(sys.argv[3])
batch = np.concatenate([pages] * (n // len(pages)))
with tempfile.TemporaryDirectory() as d:
    cm = E.Cachemap(d, 1 << 20, 12, 16)
    nh = np.full(n, 7, dtype=np.uint64); gen = np.zeros(n, dtype=np.uint32)
    cm.put_batch(np.arange(n, dtype=np.uint64) << np.uint64(16), nh, gen, batch)      # warm-up
    cm.engine_handles()
    t = time.perf_counter()
    for r in range(reps):
        cm.put_batch((np.arange(n, dtype=np.uint64) + np.uint64((r + 1) * n)) << np.uint64(16), nh, gen, batch)
    cm.engine_handles()                                    # every put is in its engine
    dt = time.perf_counter() - t
    print("PUT_BATCH_GIBS", reps * n * 65536 / dt / 2**30, len(cm.engine_handles()))
    out = np.empty_like(batch)
    t = time.perf_counter()
    for r in range(reps):
        _, hit = cm.get_batch((np.arange(n, dtype=np.uint64) + np.uint64((r + 1) * n)) << np.uint64(16), nh, gen, out=out)
    dt = time.perf_counter() - t
    assert hit.all() and (out == batch).all()
    print("GET_BATCH_GIBS", reps * n * 65536 / dt / 2**30)
    cm.free()
'''


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines() if r.returncode == 0 else ["unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", default="8,32")
    ap.add_argument("--per-thread", type=int, default=512)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--lists", default=None, help="';'-separated CMB200_DEVICES values (default: first 1..N devices)")
    a = ap.parse_args()
    ndev = E.device_count()
    if a.lists:
        lists = a.lists.split(";")
    elif ndev >= 2:
        lists = [",".join(str(i) for i in range(k)) for k in range(1, ndev + 1)]
    else:
        lists = ["0", "0,0"]
    cards = card()
    print("cards:", cards, flush=True)
    work = tempfile.mkdtemp(prefix="multidevice_bench_")
    exe = os.path.join(work, "api_threads")
    subprocess.run(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tools", "api_threads.c"), "-ldl", "-lpthread"], check=True)
    pages = np.stack([E.gen_chunk_host(42, c, 65536) for c in range(64)])
    pbin = os.path.join(work, "pages.bin")
    pages.tofile(pbin)
    lib = E.library_path()
    out = {"cards": cards, "runs": {}}
    for devs in lists:
        env = dict(os.environ, CMB200_DEVICES=devs, CMB200_PERSIST="0")
        env.setdefault("CMB200_ARENA_MB", "8192" if len(devs.split(",")) == 1 or ndev >= 2 else "4096")
        res = {}
        r = subprocess.run([sys.executable, "-c", PUT_BATCH, ROOT, pbin, str(a.batches)], capture_output=True, text=True,
                           timeout=600, env=env)
        line = [x for x in r.stdout.splitlines() if x.startswith("PUT_BATCH_GIBS")]
        res["put_batch_gibs"] = float(line[-1].split()[1]) if line else None
        gline = [x for x in r.stdout.splitlines() if x.startswith("GET_BATCH_GIBS")]
        res["get_batch_gibs"] = float(gline[-1].split()[1]) if gline else None
        if not line:
            print(devs, "put_batch failed", r.stdout[-300:], r.stderr[-300:], flush=True)
        for t in [int(x) for x in a.threads.split(",")]:
            per = min(a.per_thread, 60000 // t)
            with tempfile.TemporaryDirectory() as d:
                r = subprocess.run([exe, lib, d, pbin, str(t), str(per)], capture_output=True, text=True, timeout=300, env=env)
            line = [x for x in r.stdout.splitlines() if x.startswith("{")]
            if not line:
                print(devs, t, "failed", r.stdout[-300:], r.stderr[-300:], flush=True)
                continue
            res[f"T{t}"] = json.loads(line[-1])
        out["runs"][devs] = res
        print(devs, res, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
