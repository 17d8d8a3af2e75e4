#!/usr/bin/env python
"""Generates tests/golden/*.json from the reference itself (oracle/_ref/libcachemap_ref.so, i.e.
/root/reference/cachemap compiled unmodified, plus oracle/ref_kat.c built against the reference's
own uint128.h).  Run in the authoring container only; the fixtures it writes are committed and
are what pins the oracle (and, on the GPU box, the CUDA path) where /root/reference is absent.

    python tools/gen_golden.py [lz4 keys ref_blocks limit exerciser key_edges store]
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import datagen  # noqa: E402
from oracle import ef_oracle as O  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
REF = "/root/reference/cachemap"


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def gen_lz4():
    out = []
    for kind, n, accel, seed in datagen.codec_cases():
        page = datagen.make_page(kind, n, seed)
        blk = O.ref_lz4_encode(page, accel)
        rec = {"kind": kind, "n": n, "accel": accel, "seed": seed, "in_sha256": sha(page),
               "len": len(blk), "sha256": sha(blk)}
        if len(blk) <= 300:
            rec["hex"] = blk.hex()
        if n:
            back, used = O.ref_lz4_decode(blk, n)
            assert back == page.tobytes() and used == len(blk)
        out.append(rec)
    with open(os.path.join(GOLD, "lz4_blocks.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast of cachemap/lz4.c (v1.8.1), "
                   "called as filemap.c:126 does", "cases": out}, f, indent=0)
    print("lz4 cases:", len(out))


def gen_ref_blocks():
    """Length and SHA-256 of the reference's block for every page of the oracle's sweep and of the
    CUDA comparison, so that both comparisons run without the reference."""
    def rows(cases):
        out = []
        for kind, n, accel, seed in cases:
            page = datagen.make_page(kind, n, seed)
            blk = O.ref_lz4_encode(page, accel)
            back, used = O.ref_lz4_decode(blk, n)
            assert back == page.tobytes() and used == len(blk)
            out.append([kind, n, accel, seed, len(blk), sha(blk)[:32]])
        return out
    with open(os.path.join(GOLD, "ref_blocks.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast of cachemap/lz4.c (v1.8.1)",
                   "version": O.ref().LZ4_versionString().decode(),
                   "columns": ["kind", "n", "accel", "seed", "len", "sha256 (first 32 hex digits)"],
                   "sweep": rows(datagen.reference_sweep_cases()),
                   "gpu": rows(datagen.gpu_reference_cases())}, f, indent=0)
    print("reference blocks written")


def gen_limit():
    """The reference's LZ4_compress_fast with filemap_set's dstCapacity of n + 1024 (filemap.c:126) on
    pages whose unlimited block is within 24 bytes of that limit (pshift 18-20), plus random pages at
    pshift 17, where every block fits.  ref_len 0: the reference refused the page."""
    out = []
    for pshift in (17, 18, 19, 20):
        n = 1 << pshift
        for seed in range(3):
            for accel in (12, 1):
                base = len(O.lz4_encode(datagen.limit_page(n, 100 * pshift + seed, 0, 0), accel))
                # a zero run near the page start (where the match search still steps byte by byte)
                # shortens the block by about its length
                zlens = [0] if pshift == 17 else range(max(0, base - n - 1024 - 24), base - n - 1024 + 25, 2)
                for z in zlens:
                    at = 16 * seed
                    page = datagen.limit_page(n, 100 * pshift + seed, at, z)
                    ours = len(O.lz4_encode(page, accel))
                    if pshift > 17 and abs(ours - (n + 1024)) > 24:
                        continue
                    out.append([pshift, accel, 100 * pshift + seed, at, z, len(O.ref_lz4_encode(page, accel))])
    with open(os.path.join(GOLD, "lz4_limit.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py", "reference": "LZ4_compress_fast(page, dst, n, n + 1024, accel) "
                   "of cachemap/lz4.c (v1.8.1), called as filemap.c:126 does",
                   "columns": ["pshift", "accel", "seed", "zero_at", "zero_len", "ref_len (0: refused)"],
                   "page": "tests/datagen.py limit_page(1 << pshift, seed, zero_at, zero_len)", "cases": out}, f, indent=0)
    print("limit cases:", len(out), "refused:", sum(1 for r in out if r[-1] == 0))


def gen_exerciser(seeds=(1, 2, 3), objects=32768, pshift=15):
    """Per-phase hit counts of tests/c/exerciser.c linked against the reference's library."""
    import re
    ref = os.path.join(ROOT, "oracle", "_ref", "libcachemap_ref.so")
    exe = os.path.join(ROOT, "oracle", "_ref", "exerciser_ref")
    subprocess.run(["gcc", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c", "exerciser.c"),
                    "-o", exe, ref, f"-Wl,-rpath,{os.path.dirname(ref)}", "-lpthread"], check=True)
    runs = []
    for seed in seeds:
        for attempt in range(8):                   # the reference can hang at start-up (SURVEY.md §5)
            with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
                try:
                    out = subprocess.run([exe, d, str(objects), str(pshift), str(seed)], capture_output=True,
                                         text=True, timeout=60).stdout
                    break
                except subprocess.TimeoutExpired:
                    continue
        else:
            raise RuntimeError("the reference exerciser hung at start-up in every attempt")
        phases = {m.group(1): [int(m.group(2)), int(m.group(3))] for m in re.finditer(r"phase (\w+) hits (\d+) of (\d+)", out)}
        entries = [int(x) for x in re.findall(r"entries_after_\w+ (\d+)", out)]
        assert len(phases) == 5, out
        runs.append({"seed": seed, "phases": phases, "entries": entries})
    with open(os.path.join(GOLD, "ref_exerciser.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py: tests/c/exerciser.c linked against libcachemap_ref.so (LMDB on tmpfs)",
                   "objects": objects, "pshift": pshift, "runs": runs}, f, indent=1)
    print("exerciser runs:", runs)


def gen_keys():
    exe = os.path.join(ROOT, "oracle", "_ref", "ref_kat")
    subprocess.run(["gcc", "-O2", "-I" + REF, os.path.join(ROOT, "oracle", "ref_kat.c"), "-o", exe], check=True)
    data = json.loads(subprocess.run([exe], check=True, capture_output=True, text=True).stdout)
    data["generator"] = "oracle/ref_kat.c compiled against the reference's cachemap/uint128.h"
    with open(os.path.join(GOLD, "keys.json"), "w") as f:
        json.dump(data, f, indent=0)
    print("key KATs:", len(data["addrs"]))


def store_script(pshift=16):
    """The operation list of the store trace: C0 shape (16 x 64 KiB) plus the edge cases of
    SURVEY.md §8c.  Each op: [kind, offset, nhid, genid, content]; content = [kind, seed]."""
    import edge_fuse_b200 as E
    ops = []
    cids = list(range(16))
    off, nh = E.gen_addr(42, cids, pshift)
    for c in cids:                                   # 16 puts, config 0
        ops.append(["put", int(off[c]), int(nh[c]), 0, ["S", c]])
    for c in cids:
        ops.append(["get", int(off[c]), int(nh[c]), 0, None])
    ops.append(["put", 16 << pshift, int(nh[0]), 0, ["S", 3]])        # same content, new address
    ops.append(["get", 16 << pshift, int(nh[0]), 0, None])
    ops.append(["put", int(off[5]), int(nh[5]), 0, ["T", 999]])       # same address, new content
    ops.append(["get", int(off[5]), int(nh[5]), 0, None])
    ops.append(["get", 40 << pshift, int(nh[0]), 0, None])            # never stored
    ops.append(["get", (1 << pshift) + 1, int(nh[1]), 0, None])       # offset truncated by >> pshift
    ops.append(["get", int(off[2]), int(nh[2]), 7, None])             # other genid: miss
    ops.append(["put", int(off[2]), int(nh[2]), 7, ["Z", 5]])
    ops.append(["get", int(off[2]), int(nh[2]), 7, None])
    ops.append(["get", int(off[2]), int(nh[2]), 0, None])
    ops.append(["put", (1 << 44) << pshift, 1, 0, ["R", 1]])          # page number overflows 44 bits
    ops.append(["get", (1 << 44) << pshift, 1, 0, None])
    ops.append(["get", int(off[2]), int(nh[2]), (1 << 20) + 7, None]) # genid keeps its low 20 bits only
    ops.append(["put", int(off[9]), int(nh[9]), 0, ["R", 77]])
    ops.append(["put", int(off[9]), int(nh[9]), 0, ["M", 78]])        # twice in a row: last wins
    ops.append(["get", int(off[9]), int(nh[9]), 0, None])
    return ops


def gen_store():
    R = O.ref()
    pshift, accel = 16, 12
    ops = store_script(pshift)
    trace = []
    with tempfile.TemporaryDirectory(dir="/dev/shm" if os.path.isdir("/dev/shm") else None) as d:
        assert not R.cachemap_create(d.encode(), 1023, accel, pshift)         # n < 1024 -> NULL
        assert not R.cachemap_create((d + "/nope").encode(), 1024, accel, pshift)
        cm = R.cachemap_create(d.encode(), 1024, accel, pshift)
        assert cm
        libc = C.CDLL(None)
        libc.free.argtypes = [C.c_void_p]
        for kind, off, nh, gen, content in ops:
            if kind == "put":
                page = datagen.make_page(content[0], 1 << pshift, content[1])
                R.cachemap_put(cm, off, nh, gen, page.ctypes.data)
                trace.append(None)
            else:
                p = R.cachemap_get(cm, off, nh, gen)
                if p:
                    trace.append(sha(C.string_at(p, 1 << pshift)))
                    libc.free(p)
                else:
                    trace.append("miss")
        pages_ptr = C.cast(cm, C.POINTER(C.c_void_p))[0]                      # cm->pages
        entries = int(R.filemap_entries(pages_ptr))
        # struct cachemap tail: capacity, requests, hits are its last three u64 (cachemap.h:20-31)
        sz = 8 + 8 + 8 + 4 * 8 + 48 + 40 + 8 + 3 * 8
        raw = C.string_at(cm, sz)
        cap, req, hits = np.frombuffer(raw[-24:], dtype=np.uint64)
        assert cap == 1024, cap
        # deliberately no cachemap_free(): it can hang in the reference (SURVEY.md §5)
    with open(os.path.join(GOLD, "store_trace.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py against libcachemap_ref.so (LMDB on tmpfs)",
                   "pshift": pshift, "accel": accel, "capacity": 1024, "ops": ops, "gets": trace,
                   "entries": entries, "requests": int(req), "hits": int(hits),
                   "create_null": ["capacity 1023", "missing directory"]}, f, indent=0)
    print("store trace ops:", len(ops), "entries", entries, "requests", int(req), "hits", int(hits))
    os._exit(0)


KEY_EDGE_PSHIFTS = (12, 16, 17)         # the page sizes of the GPU replay: k_get_small 4 KiB, 64 KiB, pair 128 KiB


def key_edge_groups():
    """Addresses that share a store key (FNV-1a-64 of the 16 address bytes), found by tools/fnv_preimage.py
    from fixed seeds: a group of four, three pairs, three addresses each for the table's empty (0) and
    tombstone (~0) keys, and ordinary addresses whose keys are all different."""
    import random
    import fnv_preimage as F
    base = (0x1234, 0x100000000007)
    groups = {"quad": [base] + F.preimages(F.addr_key(*base), 3, seed=1, avoid=[base])}
    rng = random.Random(7)
    for i in range(3):
        a = (rng.getrandbits(64), rng.getrandbits(64))
        groups[f"pair{i}"] = [a] + F.preimages(F.addr_key(*a), 1, seed=10 + i, avoid=[a])
    groups["key0"] = F.preimages(0, 3, seed=20)
    groups["key_ones"] = F.preimages(F.MASK, 3, seed=21)
    ordinary = [(rng.getrandbits(64), rng.getrandbits(64)) for _ in range(6)]
    keys = [F.addr_key(*a) for a in ordinary] + [F.addr_key(*g[0]) for g in groups.values()]
    assert len(set(keys)) == len(keys)
    for g in groups.values():
        assert len(set(g)) == len(g) and len({F.addr_key(*a) for a in g}) == 1
    return groups, ordinary


def key_edge_script(groups, ordinary):
    """Ops [kind, u, l, content]: per group (members A, B, C...) put A, get A, put B, get A, get B; put A
    again, get B, get A; unset through C (B for a pair), get every member; put B again, get B, get A —
    with an ordinary address put and read around each group."""
    kinds = "TMRXZ"
    ops, seed = [], [0]

    def put(a):
        seed[0] += 1
        ops.append(["put", a[0], a[1], [kinds[seed[0] % len(kinds)], seed[0]]])

    def get(a):
        ops.append(["get", a[0], a[1], None])

    for gi, g in enumerate(groups.values()):
        A, B = g[0], g[1]
        C = g[2] if len(g) > 2 else B
        o = ordinary[gi % len(ordinary)]
        put(o)
        put(A); get(A); put(B); get(A); get(B)
        get(o)
        put(A); get(B); get(A)
        ops.append(["unset", C[0], C[1], None])
        for a in g:
            get(a)
        get(o)
        put(B); get(B); get(A)
    for o in ordinary:
        get(o)
    return ops


def _key_edges_ref(pshift: str, ops_path: str, destdir: str):
    """Child process of gen_key_edges: replays the ops against the reference, writing after each op
    (and after the reference's own stdout has been flushed) `op <i> <answer>`, then one JSON line."""
    pshift = int(pshift)
    R = O.ref()
    R.filemap_unset.restype = None
    R.filemap_unset.argtypes = [C.c_void_p, C.c_void_p]
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    libc.fflush.argtypes = [C.c_void_p]
    with open(ops_path) as f:
        ops = json.load(f)
    cm = R.cachemap_create(destdir.encode(), 1024, 12, pshift)
    assert cm
    pages_ptr = C.cast(cm, C.POINTER(C.c_void_p))[0]                          # cm->pages
    for i, (kind, u, l, content) in enumerate(ops):
        off, gen = (l & ((1 << 44) - 1)) << pshift, l >> 44
        ans = "-"
        if kind == "put":
            page = datagen.make_page(content[0], 1 << pshift, content[1])
            R.cachemap_put(cm, off, u, gen, page.ctypes.data)
        elif kind == "unset":
            R.filemap_unset(pages_ptr, (C.c_uint64 * 2)(u, l))
        else:
            p = R.cachemap_get(cm, off, u, gen)
            ans = sha(C.string_at(p, 1 << pshift)) if p else "miss"
            if p:
                libc.free(p)
        libc.fflush(None)
        os.write(1, f"op {i} {ans}\n".encode())
    entries = int(R.filemap_entries(pages_ptr))
    sz = 8 + 8 + 8 + 4 * 8 + 48 + 40 + 8 + 3 * 8                               # as in gen_store
    _, req, hits = np.frombuffer(C.string_at(cm, sz)[-24:], dtype=np.uint64)
    libc.fflush(None)
    os.write(1, (json.dumps({"entries": entries, "requests": int(req), "hits": int(hits)}) + "\n").encode())
    os._exit(0)                             # no cachemap_free(): it can hang in the reference (SURVEY.md §5)


def gen_key_edges():
    """tests/golden/key_edges.json: colliding and sentinel-key addresses and the reference's answers to a
    trace over them at every page size of KEY_EDGE_PSHIFTS.  Each get's answer is the SHA-256 of the page,
    "miss", or "bad entry" when the reference printed `bad entry` for it (filemap.c:237)."""
    import re
    import shutil
    groups, ordinary = key_edge_groups()
    ops = key_edge_script(groups, ordinary)
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        ops_path = os.path.join(tmp, "ops.json")
        with open(ops_path, "w") as f:
            json.dump(ops, f)
        for pshift in KEY_EDGE_PSHIFTS:
            for attempt in range(8):                    # the reference can hang at start-up (SURVEY.md §5)
                d = tempfile.mkdtemp(dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
                try:
                    out = subprocess.run([sys.executable, os.path.abspath(__file__), "_key_edges_ref", str(pshift),
                                          ops_path, d], capture_output=True, text=True, timeout=120).stdout
                    break
                except subprocess.TimeoutExpired:
                    continue
                finally:
                    shutil.rmtree(d, ignore_errors=True)
            else:
                raise RuntimeError("the reference hung in every attempt")
            lines = out.splitlines()
            tail = json.loads(lines[-1])
            gets, bad_since = [], 0
            for line in lines[:-1]:
                if line == "bad entry":
                    bad_since += 1
                    continue
                m = re.fullmatch(r"op (\d+) (\S+)", line)
                assert m, line
                i, ans = int(m.group(1)), m.group(2)
                assert bad_since <= (ops[i][0] == "get" and ans == "miss"), (i, ans, bad_since)
                if ops[i][0] == "get":
                    gets.append("bad entry" if bad_since else ans)
                bad_since = 0
            assert len(gets) == sum(op[0] == "get" for op in ops)
            runs[str(pshift)] = {"gets": gets, "bad_entries": gets.count("bad entry"), **tail}
    with open(os.path.join(GOLD, "key_edges.json"), "w") as f:
        json.dump({"generator": "tools/gen_golden.py key_edges (addresses: tools/fnv_preimage.py) against "
                   "libcachemap_ref.so (LMDB on tmpfs): cachemap_put, cachemap_get, filemap_unset",
                   "capacity": 1024, "accel": 12,
                   "op": "[kind, u, l, content]: offset = (l & (2^44 - 1)) << pshift, nhid = u, genid = l >> 44; "
                         "content = datagen.make_page(content[0], 1 << pshift, content[1])",
                   "groups": {k: [list(a) for a in v] for k, v in groups.items()},
                   "ordinary": [list(a) for a in ordinary], "ops": ops, "runs": runs}, f, indent=0)
    print("key edges ops:", len(ops), {p: {k: v for k, v in r.items() if k != "gets"} for p, r in runs.items()})


if __name__ == "__main__":
    if sys.argv[1:2] == ["_key_edges_ref"]:
        _key_edges_ref(*sys.argv[2:])
    assert O.ref() is not None, "oracle/_ref/libcachemap_ref.so missing: run make -C oracle"
    os.makedirs(GOLD, exist_ok=True)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    steps = {"lz4": gen_lz4, "keys": gen_keys, "ref_blocks": gen_ref_blocks, "limit": gen_limit, "exerciser": gen_exerciser,
             "key_edges": gen_key_edges, "store": gen_store}   # gen_store ends the process: keep it last
    for name in sys.argv[1:] or steps:
        steps[name]()
