#!/usr/bin/env python
"""What encryption at rest costs (DESIGN.md §2 "Encryption at rest").  One JSON line with:
  - card: the GPU's name, power limit and max SM clock, read in the same call;
  - kernels: k_seal and k_open time (torch.profiler, CUDA activities) over batches of record-sized
    messages (4 KiB, 64 KiB and 1 MiB pages' records) through cmb200_aead_seal_batch / _open_batch, their
    GB/s, and the integer bound: INT32 lanes x SMs x max SM clock over the instructions per byte the
    kernels need (OPS_PER_BYTE below, counted from aead.cuh);
  - save / load: wall time of cmb200_save_set and cmb200_load_chain of --gib GiB of records of the
    synthetic stream's R and T pages at 64 KiB and 4 KiB, without and with a key, alternated --rounds times;
  - put stall: per-call latency of back-to-back 256-page puts while the store is saved, without and with
    a key (as tools/snapshot_bench.py measures it), 64 KiB pages.
Files go under --dir and are removed.

    python tools/crypt_bench.py --dir /tmp/cryptbench --gib 8 --rounds 2
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

GIB = 1 << 30
KEY = bytes(range(0x11, 0x31))
# ChaCha20: 80 quarter rounds x 12 instructions + 32 (feed-forward, xor) per 64 bytes = 15.5 / byte;
# Poly1305: 25 32x32->64 multiply-adds (2 issue slots each) + ~30 carries, masks and adds per 16 bytes = 5 / byte
OPS_PER_BYTE = 15.5 + 5.0
INT32_LANES_PER_SM = 64


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,count", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock, _n = [x.strip() for x in q[0].split(",")]
    return {"name": name, "power_limit_w": float(power), "max_sm_mhz": float(clock)}


def kernels(E, card):
    import torch
    from torch.profiler import ProfilerActivity, profile
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bound = INT32_LANES_PER_SM * sms * card["max_sm_mhz"] * 1e6 / OPS_PER_BYTE / 1e9
    out = {"sms": sms, "int_bound_gbs": bound, "ops_per_byte": OPS_PER_BYTE, "sizes": {}}
    rng = np.random.default_rng(1)
    for label, size, n in (("4k", 24 + 4096 + 8, 16384), ("64k", 24 + 65536 + 8, 2048), ("1m", 24 + (1 << 20) + 8, 128)):
        msgs = [rng.integers(0, 256, size, dtype=np.uint8).tobytes() for _ in range(n)]
        aads = [bytes(24)] * n
        nonces = [i.to_bytes(12, "little") for i in range(n)]
        sealed = E.aead_seal_batch(KEY, nonces, aads, msgs)          # warm-up
        assert E.aead_open_batch(KEY, nonces[:4], aads[:4], sealed[:4]) == msgs[:4]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                E.aead_seal_batch(KEY, nonces, aads, msgs)
                E.aead_open_batch(KEY, nonces, aads, sealed)
        t = {}
        for ev in prof.key_averages():
            for k in ("k_seal", "k_open"):
                if k in ev.key and ev.count:
                    t[k] = t.get(k, 0.0) + ev.device_time_total / ev.count * 1e-6
        row = {"n": n, "bytes": n * size}
        for k, s in t.items():
            row[k + "_ms"] = s * 1e3
            row[k + "_gbs"] = n * size / s / 1e9
        out["sizes"][label] = row
    return out


def _pool(E, bs, n=512):
    # cid % 4 == 0: R (incompressible), 1: T (text-like), as tools/snapshot_bench.py uses them
    return np.stack([E.gen_chunk_host(42, 4 * (c // 2) + (c % 2), bs) for c in range(n)])


def _fill(E, eng, pool, nh, target):
    big = np.concatenate([pool] * max(1, 4096 // len(pool)))
    n = 0
    while eng.stats()["arena_used"] < target:
        eng.put(np.full(len(big), nh, dtype=np.uint64), np.arange(n, n + len(big), dtype=np.uint64), big)
        n += len(big)
    return n


def _pct(xs):
    xs = np.sort(np.asarray(xs))
    return {"n": int(len(xs)), "p50_ms": float(np.percentile(xs, 50) * 1e3), "p99_ms": float(np.percentile(xs, 99) * 1e3),
            "max_ms": float(xs[-1] * 1e3)}


def save_load(E, a, pshift):
    bs = 1 << pshift
    target = int(a.gib * GIB)
    cap = 2 * target // min(bs, 2048) + 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=cap, arena_bytes=target + (2 << 30), max_batch=4096,
                   flags=E.FINGERPRINT)
    recs = _fill(E, eng, _pool(E, bs), 1, target)
    path = os.path.join(a.dir, f"crypt_{pshift}.snap")
    out = {"records": recs, "arena_gib": eng.stats()["arena_used"] / GIB, "save": {"plain": [], "key": []},
           "load": {"plain": [], "key": []}}
    for _r in range(a.rounds):
        for mode in ("plain", "key"):
            eng.set_file_key(KEY if mode == "key" else None)
            t0 = time.perf_counter()
            n = E.save_set([eng.h], path)
            el = time.perf_counter() - t0
            size = os.path.getsize(path)
            out["save"][mode].append({"s": el, "file_gib": size / GIB, "gibs": size / GIB / el, "records": n})
            dst = E.Engine(pshift=pshift, accel=12, capacity=cap, arena_bytes=target + (2 << 30), max_batch=4096,
                           flags=E.FINGERPRINT)
            dst.set_file_key(KEY if mode == "key" else None)
            t0 = time.perf_counter()
            got, _k = E.load_chain([dst.h], path)
            el = time.perf_counter() - t0
            out["load"][mode].append({"s": el, "gibs": size / GIB / el, "records": got, "rejected": dst.load_rejected()})
            assert got == n
            dst.close()
            os.remove(path)
    eng.close()
    return out


def put_stall(E, a):
    bs = 65536
    target = int(a.gib * GIB)
    pool = _pool(E, bs)
    eng = E.Engine(pshift=16, accel=12, capacity=1 << 20, arena_bytes=target + (16 << 30), max_batch=4096)
    _fill(E, eng, pool, 1, target)
    path = os.path.join(a.dir, "stall.snap")
    u = np.full(256, 2, dtype=np.uint64)
    l = np.arange(256, dtype=np.uint64)
    batch = np.ascontiguousarray(pool[:256])
    eng.put(u, l, batch)
    out = {}
    for _r in range(a.rounds):
        for mode in ("plain", "key"):
            eng.set_file_key(KEY if mode == "key" else None)
            eng.compact()
            res = {}

            def save():
                t0 = time.perf_counter()
                E.save_set([eng.h], path)
                res["save_s"] = time.perf_counter() - t0

            th = threading.Thread(target=save)
            lat = []
            th.start()
            while th.is_alive() or len(lat) < 20:
                t0 = time.perf_counter()
                eng.put(u, l, batch)
                lat.append(time.perf_counter() - t0)
            th.join()
            os.remove(path)
            out.setdefault(mode, []).append(dict(_pct(lat), **res))
    lat = []
    for _ in range(200):
        t0 = time.perf_counter()
        eng.put(u, l, batch)
        lat.append(time.perf_counter() - t0)
    out["no_save"] = _pct(lat)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True)
    ap.add_argument("--gib", type=float, default=8.0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip", default="", help="comma list of parts to leave out: kernels,save64k,save4k,stall")
    a = ap.parse_args()
    os.makedirs(a.dir, exist_ok=True)
    import edge_fuse_b200 as E
    skip = set(a.skip.split(","))
    card = _card()
    line = {"card": card, "gib": a.gib, "rounds": a.rounds}
    try:
        if "kernels" not in skip:
            line["kernels"] = kernels(E, card)
        if "save64k" not in skip:
            line["save_load_64k"] = save_load(E, a, 16)
        if "save4k" not in skip:
            line["save_load_4k"] = save_load(E, a, 12)
        if "stall" not in skip:
            line["put_stall_64k"] = put_stall(E, a)
    finally:
        shutil.rmtree(a.dir, ignore_errors=True)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
