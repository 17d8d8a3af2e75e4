#!/usr/bin/env python
"""What a snapshot costs the store that is being saved.  Each library runs in a subprocess of its own
(CMB200_LIB), so that two builds can alternate in one call:

    python tools/snapshot_bench.py --dir /dev/shm/snapbench --lib new=edge_fuse_b200/libcachemap.so.0.0 \\
        --lib old=/path/to/other/tree/edge_fuse_b200/libcachemap.so.0.0 --rounds 2

(each library is driven by the Python binding of the tree it was built in).

Per library and round, with 64 KiB pages (pshift 16) of the synthetic stream's R and T classes:
  - save rate: wall time of cmb200_save of a store of --gib GiB of records and the file's GiB/s, for an
    engine without a host tier and for one whose records are half in the tier;
  - put stall: per-call latency of back-to-back 256-page cmb200_put_batch calls from one thread, without
    a save and while another thread saves the store (p50, p99, max);
  - compaction wait: time spent in cmb200_compact called 50 ms after a save started;
  - a small store of single-page puts (deterministic record order) saved to <dir>/cmp_<name>_<round>.snap,
    whose bytes must be the same for every library.
Then the drop-in: cachemap_put of 64 KiB pages from 8 native threads for --dropin-sec seconds, with
CMB200_CHECKPOINT_SEC=1 and without it (tools/checkpoint_puts.c).  The card's name and power limit are
read in the same call.  Files go under --dir (tmpfs takes the disk out).  Prints one JSON line."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

GIB = 1 << 30
BS = 65536


def _pool(E, n=512):
    # cid % 4 == 0: R (incompressible), 1: T (text-like) in the synthetic stream's class layout
    return np.stack([E.gen_chunk_host(42, 4 * (c // 2) + (c % 2), BS) for c in range(n)])


def _pct(xs):
    xs = np.sort(np.asarray(xs))
    return {"n": int(len(xs)), "p50_ms": float(np.percentile(xs, 50) * 1e3), "p99_ms": float(np.percentile(xs, 99) * 1e3),
            "max_ms": float(xs[-1] * 1e3)}


def _fill(E, eng, pool, nh, first, target_bytes):
    """Puts distinct keys (nh, first + i) until the store's records reach target_bytes -> keys put."""
    big = np.concatenate([pool] * 8)
    n = 0
    while eng.stats()["arena_used"] < target_bytes:
        l = np.arange(first + n, first + n + len(big), dtype=np.uint64)
        eng.put(np.full(len(big), nh, dtype=np.uint64), l, big)
        n += len(big)
    return n


def _timed_save(eng, path):
    t0 = time.perf_counter()
    recs = eng.save(path)
    el = time.perf_counter() - t0
    size = os.path.getsize(path)
    os.remove(path)
    return {"s": el, "records": int(recs), "gib": size / GIB, "gibs": size / GIB / el}


def child(a):
    # the binding of the library's own tree (<tree>/edge_fuse_b200/libcachemap.so.0.0)
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.environ["CMB200_LIB"])))
    import edge_fuse_b200 as E
    pool = _pool(E)
    out = {}
    # a store of single-page puts: every record's arena offset follows from the call order
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=1 << 30, max_batch=64, flags=E.FINGERPRINT,
                   host_tier_bytes=256 << 20)
    for i in range(1024):
        eng.put(np.array([7], dtype=np.uint64), np.array([i], dtype=np.uint64), pool[i % len(pool)][None],
                ts=np.array([1000 + i], dtype=np.uint64))
    eng.demote(np.full(256, 7, dtype=np.uint64), np.arange(256, dtype=np.uint64))
    eng.save(a.cmp_file)
    eng.close()

    target = int(a.gib * GIB)
    # no tier: room for the store plus the puts made while it is saved
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 20, arena_bytes=target + (24 << 30), max_batch=4096)
    _fill(E, eng, pool, 1, 0, target)
    path = os.path.join(a.dir, f"bench_{os.getpid()}.snap")
    out["save_no_tier"] = _timed_save(eng, path)
    u = np.full(256, 2, dtype=np.uint64)
    l = np.arange(256, dtype=np.uint64)
    batch = np.ascontiguousarray(pool[:256])
    eng.put(u, l, batch)
    lat = []
    for _ in range(200):
        t0 = time.perf_counter()
        eng.put(u, l, batch)
        lat.append(time.perf_counter() - t0)
    out["put_no_save"] = _pct(lat)
    eng.compact()
    res = {}
    th = threading.Thread(target=lambda: res.update(_timed_save(eng, path)))
    lat = []
    th.start()
    while th.is_alive() or len(lat) < 20:
        t0 = time.perf_counter()
        eng.put(u, l, batch)
        lat.append(time.perf_counter() - t0)
    th.join()
    out["put_during_save"] = _pct(lat)
    out["save_during_puts"] = res
    eng.compact()
    res = {}
    th = threading.Thread(target=lambda: res.update(_timed_save(eng, path)))
    th.start()
    time.sleep(0.05)
    t0 = time.perf_counter()
    eng.compact()
    out["compact_after_save_start_s"] = time.perf_counter() - t0
    th.join()
    out["save_with_compact"] = res
    eng.close()

    # half of the records in the host tier
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 20, arena_bytes=target // 2 + (2 << 30), max_batch=4096,
                   host_tier_bytes=target // 2 + (1 << 30))
    n = _fill(E, eng, pool, 3, 0, target // 2)
    for base in range(0, n, 65536):
        m = min(65536, n - base)
        eng.demote(np.full(m, 3, dtype=np.uint64), np.arange(base, base + m, dtype=np.uint64))
    eng.compact()
    _fill(E, eng, pool, 3, n, target - E.host_tier_stats(eng.h)["used"])
    out["tier_used_gib"] = E.host_tier_stats(eng.h)["used"] / GIB
    out["save_half_tier"] = _timed_save(eng, path)
    eng.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True, help="where the snapshot files go (tmpfs takes the disk out)")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="a library to measure (repeatable)")
    ap.add_argument("--gib", type=float, default=8.0)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--dropin-sec", type=float, default=10.0)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--cmp-file", help=argparse.SUPPRESS)
    a = ap.parse_args()
    os.makedirs(a.dir, exist_ok=True)
    if a.child:
        return child(a)
    import edge_fuse_b200 as E
    libs = [x.split("=", 1) for x in a.lib] or [["this", E.library_path()]]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    line = {"card": smi[0] if smi else "unknown", "dir": a.dir, "gib": a.gib, "runs": {}, "dropin": {}}
    cmp_files = []
    for r in range(a.rounds):
        for name, lib in libs:
            cf = os.path.join(a.dir, f"cmp_{name}_{r}.snap")
            env = dict(os.environ, CMB200_LIB=os.path.abspath(lib))
            p = subprocess.run([sys.executable, __file__, "--child", "--dir", a.dir, "--gib", str(a.gib), "--cmp-file", cf],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                line["runs"].setdefault(name, []).append({"error": p.stderr[-2000:]})
                continue
            line["runs"].setdefault(name, []).append(json.loads(p.stdout.strip().splitlines()[-1]))
            cmp_files.append(cf)
    if len(cmp_files) > 1:
        line["cmp_identical"] = all(subprocess.run(["cmp", "-s", cmp_files[0], f]).returncode == 0 for f in cmp_files[1:])
    for f in cmp_files:
        os.remove(f)
    work = tempfile.mkdtemp(prefix="checkpoint_puts_")
    exe = os.path.join(work, "checkpoint_puts")
    subprocess.run(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tools", "checkpoint_puts.c"), "-ldl", "-lpthread"], check=True)
    pbin = os.path.join(work, "pages.bin")
    _pool(E, 64).tofile(pbin)
    for r in range(a.rounds):
        for name, lib in libs:
            for sec in ("1", "0"):
                d = tempfile.mkdtemp(dir=a.dir)
                env = dict(os.environ, CMB200_CHECKPOINT_SEC=sec, CMB200_PERSIST="1", CMB200_ARENA_MB="8192")
                p = subprocess.run([exe, os.path.abspath(lib), d, pbin, "8", str(a.dropin_sec)], env=env,
                                   capture_output=True, text=True)
                res = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else {"error": p.stderr[-2000:]}
                line["dropin"].setdefault(f"{name}_checkpoint_{sec}", []).append(res)
                shutil.rmtree(d, ignore_errors=True)
    shutil.rmtree(work, ignore_errors=True)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
