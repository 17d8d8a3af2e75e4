#!/usr/bin/env python
"""Per-chunk timeline of one bench-shaped k_encode launch (16 384 x 64 KiB chunks, pages in HBM,
fingerprint on, accel 12): which warp slot encoded each chunk, and when it started and ended
(%globaltimer).  From it: per-class chunk durations, the idle warp-time fraction of the launch and its
tail (first warp out of work -> end of the launch).  Two inputs: the bench's synthetic stream (seed 42,
class from the chunk id, for reporting only) and 64 KiB pages cut from the files of this tree (the
built libraries, and the .cu/.cuh/.py/.md sources of the top level, edge_fuse_b200, include,
oracle, tests and tools), repeated to fill the launch.

Needs a library built with the timeline compiled in, selected with CMB200_LIB:

    python tools/build_variant.py timeline -DCMB_ENC_TIMELINE
    CMB200_LIB=edge_fuse_b200/build/variants/timeline.so python tools/encode_timeline.py --label new --out DIR

Prints one JSON line per input; --out DIR also gets the per-chunk arrays (<label>_<input>.npz).
With a library that has the longest-first handout, the sample statistics of k_cost come along
(starts, match-less positions, bucket), and k_cost's own time is taken with torch.profiler.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import edge_fuse_b200 as E  # noqa: E402

CHUNK, PSHIFT, ACCEL, SEED = 65536, 16, 12, 42
CLASSES = "RTZM"


def tree_pages(n: int):
    """n pages cut from this tree's libraries and sources (each kind concatenated, then cut), cycled:
    the files at the top of the tree and under the project's own directories (build directories and
    the tuning variants in them left out)."""
    libs, srcs = [], []
    walk = [(ROOT, [], sorted(f for f in os.listdir(ROOT) if os.path.isfile(os.path.join(ROOT, f))))]
    for top in ("edge_fuse_b200", "include", "oracle", "tests", "tools"):
        walk += list(os.walk(os.path.join(ROOT, top)))
    for dp, dn, fn in walk:
        if any(part.startswith("build") for part in os.path.relpath(dp, ROOT).split(os.sep)):
            continue
        for f in sorted(fn):
            if ".so" in f:
                libs.append(os.path.join(dp, f))
            elif f.endswith((".cu", ".cuh", ".py", ".md")):
                srcs.append(os.path.join(dp, f))
    pages, kinds = [], []
    for kind, paths in (("lib", libs), ("src", srcs)):
        blob = np.concatenate([np.fromfile(p, dtype=np.uint8) for p in paths])
        k = len(blob) // CHUNK
        pages.append(blob[: k * CHUNK].reshape(k, CHUNK))
        kinds += [kind] * k
    pages, kinds = np.concatenate(pages), np.array(kinds)
    pick = np.arange(n) % len(pages)
    return np.ascontiguousarray(pages[pick]), kinds[pick], len(pages)


def analyse(rec: np.ndarray, cls: np.ndarray) -> dict:
    gw, t0, t1, est = rec[:, 0], rec[:, 1].astype(np.int64), rec[:, 2].astype(np.int64), rec[:, 3]
    assert (t0 > 0).all() and (t1 >= t0).all(), "a chunk has no timeline entry"
    start, end = int(t0.min()), int(t1.max())
    span = end - start
    dur = (t1 - t0) / 1e3
    slots = np.unique(gw)
    last_end = np.array([t1[gw == w].max() for w in slots])
    busy = float((t1 - t0).sum())
    out = {"launch_us": span / 1e3, "warp_slots": int(len(slots)), "chunks_per_slot": len(rec) / len(slots),
           "idle_warp_time_frac": 1.0 - busy / (len(slots) * span),
           "tail_us": (end - int(last_end.min())) / 1e3,
           "tail_frac": (end - int(last_end.min())) / span, "classes": {}}
    starts, lits, bucket = (est >> np.uint64(16)) & np.uint64(0xFFFF), est & np.uint64(0xFFFF), est >> np.uint64(32)
    for c in np.unique(cls):
        m = cls == c
        d = {"chunks": int(m.sum()), "mean_us": float(dur[m].mean()), "std_us": float(dur[m].std()),
             "p5_us": float(np.percentile(dur[m], 5)), "p95_us": float(np.percentile(dur[m], 95))}
        if est.any():
            d.update({"sample_starts": float(starts[m].mean()), "sample_matchless": float(lits[m].mean()),
                      "buckets": np.bincount(bucket[m].astype(np.int64), minlength=8).tolist()})
        out["classes"][str(c)] = d
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--label", default="lib")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=16384)
    ap.add_argument("--out", help="directory for the per-chunk arrays")
    a = ap.parse_args()
    n = a.chunks
    L = E.lib()
    if not hasattr(L, "cmb200_enc_timeline"):
        sys.exit(f"{E.library_path()} has no encoder timeline: build it with -DCMB_ENC_TIMELINE (tools/build_variant.py)")
    tl_set = L.cmb200_enc_timeline
    tl_set.argtypes, tl_set.restype = [C.c_void_p], C.c_int
    import torch
    # the bench's arena geometry: 2 MiB segments per warp slot (engine.cu, direct encode)
    eng = E.Engine(pshift=PSHIFT, accel=ACCEL, capacity=4 * n * (a.reps + 2), arena_bytes=32 << 30, max_batch=n,
                   flags=E.FINGERPRINT)
    d_pages = eng.dev_alloc(n * CHUNK)
    d_tl = eng.dev_alloc(n * 32)
    zero = np.zeros(n * 4, dtype=np.uint64)
    cids = np.arange(n, dtype=np.uint64)
    off, nh = E.gen_addr(SEED, cids, PSHIFT)
    page_no = off >> np.uint64(PSHIFT)
    gen = [0]

    def put():
        gen[0] += 1
        return eng.put(nh, page_no | (np.uint64(gen[0]) << np.uint64(44)), d_pages, on_dev=True)

    for name in ("synthetic", "tree_files"):
        if name == "synthetic":
            eng.gen_chunks_dev(SEED, cids, d_pages)
            cls = np.array([CLASSES[c] for c in ((cids + (cids >> np.uint64(3))) & np.uint64(3)).astype(np.int64)])
            distinct = n
        else:
            pages, cls, distinct = tree_pages(n)
            eng.h2d(d_pages, pages)
            del pages
        _check(tl_set(None))
        put()                                                     # warm-up
        runs, recs = [], []
        for _ in range(a.reps):
            eng.h2d(d_tl, zero)
            _check(tl_set(C.c_void_p(d_tl)))
            s0 = eng.stats()
            put()
            s1 = eng.stats()
            _check(tl_set(None))
            rec = np.zeros((n, 4), dtype=np.uint64)
            eng.d2h(rec, d_tl)
            r = analyse(rec, cls)
            r["encode_event_us"] = (s1["encode_kernel_ns"] - s0["encode_kernel_ns"]) / 1e3
            runs.append(r)
            recs.append(rec)
        # kernel times without the timeline, in a run of their own
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            put()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            for k in ("k_cost", "k_encode", "k_upsert"):
                if k in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                    kern[k] = kern.get(k, 0.0) + ev.device_time_total
        line = {"label": a.label, "input": name, "chunks": n, "distinct_pages": int(distinct),
                "lib": os.path.relpath(E.library_path(), ROOT), "gpu": torch.cuda.get_device_name(0),
                "kernel_us_profiler": kern,
                "idle_warp_time_frac": [r["idle_warp_time_frac"] for r in runs],
                "tail_us": [r["tail_us"] for r in runs],
                "launch_us": [r["launch_us"] for r in runs],
                "encode_event_us": [r["encode_event_us"] for r in runs],
                "last_run": runs[-1]}
        print(json.dumps(line), flush=True)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            np.savez_compressed(os.path.join(a.out, f"{a.label}_{name}.npz"), rec=np.stack(recs), cls=cls)
    eng.close()


def _check(rc):
    if rc != 0:
        raise RuntimeError(f"cmb200_enc_timeline failed: {E.last_error()}")


if __name__ == "__main__":
    main()
