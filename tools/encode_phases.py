#!/usr/bin/env python
"""Where the cycles of the LZ4 parse loop go: one bench-shaped k_encode launch (16 384 x 64 KiB chunks
of the bench stream, seed 42, pages in HBM, fingerprint on, accel 12) with lane 0 of every fourth
resident warp slot stamping clock64() at fixed points of each iteration of lz4_encode_lean
(lz4_encode_ring.cuh, ENC_PH_*).  Per chunk class (R/T/Z/M, from the chunk id as in the generator)
it reports SM cycles per loop iteration by phase, how often each phase ran per iteration, and the
card's name and power limit.

Needs a library built with the phase clocks compiled in, selected with CMB200_LIB:

    python tools/build_variant.py phases -DCMB_ENC_PHASES
    CMB200_LIB=edge_fuse_b200/build/variants/phases.so python tools/encode_phases.py --label new

The stamps themselves cost a few instructions each, so absolute figures are a little above the
product build's; compare builds with the same instrumentation.  Prints one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import edge_fuse_b200 as E  # noqa: E402

CHUNK, PSHIFT, ACCEL, SEED = 65536, 16, 12, 42
CLASSES = "RTZM"
PHASES = ["head", "events", "table", "emit", "wait", "resolve", "search_slow", "count_long", "catchup_long",
          "emit_general"]


def card() -> dict:
    import torch
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q[0].split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--label", default="lib")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=16384)
    a = ap.parse_args()
    n = a.chunks
    L = E.lib()
    if not hasattr(L, "cmb200_enc_phases"):
        sys.exit(f"{E.library_path()} has no phase clocks: build it with -DCMB_ENC_PHASES (tools/build_variant.py)")
    ph_set = L.cmb200_enc_phases
    ph_set.argtypes, ph_set.restype = [C.c_void_p, C.POINTER(C.c_uint32)], C.c_int
    nph = C.c_uint32(0)
    _check(ph_set(None, C.byref(nph)))
    assert nph.value == len(PHASES), f"the library has {nph.value} phases, this tool knows {len(PHASES)}"
    P = nph.value
    eng = E.Engine(pshift=PSHIFT, accel=ACCEL, capacity=4 * n * (a.reps + 2), arena_bytes=32 << 30, max_batch=n,
                   flags=E.FINGERPRINT)
    d_pages = eng.dev_alloc(n * CHUNK)
    d_ph = eng.dev_alloc(n * 2 * P * 8)
    zero = np.zeros(n * 2 * P, dtype=np.uint64)
    cids = np.arange(n, dtype=np.uint64)
    off, nh = E.gen_addr(SEED, cids, PSHIFT)
    page_no = off >> np.uint64(PSHIFT)
    cls = np.array([CLASSES[c] for c in ((cids + (cids >> np.uint64(3))) & np.uint64(3)).astype(np.int64)])
    eng.gen_chunks_dev(SEED, cids, d_pages)
    gen = [0]

    def put():
        gen[0] += 1
        return eng.put(nh, page_no | (np.uint64(gen[0]) << np.uint64(44)), d_pages, on_dev=True)

    put()                                                         # warm-up, clocks off
    runs = []
    for _ in range(a.reps):
        eng.h2d(d_ph, zero)
        _check(ph_set(C.c_void_p(d_ph), None))
        s0 = eng.stats()
        put()
        s1 = eng.stats()
        _check(ph_set(None, None))
        rec = np.zeros((n, 2, P), dtype=np.uint64)
        eng.d2h(rec, d_ph)
        by = {}
        for c in CLASSES:
            m = (cls == c) & (rec[:, 1, PHASES.index("table")] > 0)   # sampled chunks of this class
            cyc, cnt = rec[m, 0, :].sum(axis=0).astype(np.float64), rec[m, 1, :].sum(axis=0).astype(np.float64)
            iters = cnt[PHASES.index("table")]
            if not m.any() or iters == 0:
                continue
            by[c] = {"chunks": int(m.sum()), "iters_per_chunk": iters / m.sum(),
                     "cycles_per_iter": float(cyc.sum() / iters),
                     "phase_cycles_per_iter": {p: round(float(cyc[k] / iters), 1) for k, p in enumerate(PHASES)},
                     "phase_runs_per_iter": {p: round(float(cnt[k] / iters), 4) for k, p in enumerate(PHASES)}}
        runs.append({"encode_event_us": (s1["encode_kernel_ns"] - s0["encode_kernel_ns"]) / 1e3, "classes": by})
    line = {"label": a.label, "chunks": n, "lib": os.path.relpath(E.library_path(), ROOT), **card(),
            "encode_event_us": [r["encode_event_us"] for r in runs],
            "T_cycles_per_iter": [r["classes"].get("T", {}).get("cycles_per_iter") for r in runs],
            "last_run": runs[-1]}
    print(json.dumps(line), flush=True)
    eng.close()


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"cmb200_enc_phases failed: {E.last_error()}")


if __name__ == "__main__":
    main()
