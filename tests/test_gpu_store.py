"""GPU parity, store level: hit/miss decisions, stored records and counters of the CUDA cachemap
against the reference trace fixture and the oracle's store model, through the drop-in C API."""
import hashlib
import json
import os
import threading

import numpy as np
import pytest

import datagen

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(autouse=True)
def small_engine(monkeypatch):
    monkeypatch.setenv("CMB200_ARENA_MB", "512")
    monkeypatch.setenv("CMB200_MAX_BATCH", "512")
    monkeypatch.setenv("CMB200_FINGERPRINT", "1")


def test_reference_trace_through_cachemap_api(E, gpu, tmp_path):
    """config 0 of BASELINE.json: 16 x 64 KiB + the edge cases, one call per page, same calls the
    reference answered when tools/gen_golden.py recorded the fixture."""
    t = json.load(open(os.path.join(GOLD, "store_trace.json")))
    assert not E.Cachemap(str(tmp_path), 1023, t["accel"], t["pshift"]).ok
    assert not E.Cachemap(str(tmp_path / "nope"), 1024, t["accel"], t["pshift"]).ok
    cm = E.Cachemap(str(tmp_path), t["capacity"], t["accel"], t["pshift"])
    assert cm.ok
    gets = []
    for kind, off, nh, gen, content in t["ops"]:
        if kind == "put":
            cm.put(off, nh, gen, datagen.make_page(content[0], cm.bsize, content[1]))
            gets.append(None)
        else:
            p = cm.get(off, nh, gen)
            gets.append("miss" if p is None else sha(p))
    assert gets == t["gets"]
    assert cm.counters() == (t["requests"], t["hits"])
    assert E.lib().filemap_entries(_pages_ptr(cm)) == t["entries"]
    cm.free()


def _pages_ptr(cm):
    import ctypes
    return ctypes.cast(cm.h, ctypes.POINTER(ctypes.c_void_p))[0]       # struct cachemap { pages, ...


def test_records_are_the_references_bytes(E, gpu, oracle):
    """What sits in the arena for an address is byte for byte the LMDB value of the reference:
    24-byte data_prefix + LZ4 block (filemap.c:140-147)."""
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=256 << 20, max_batch=256,
                   flags=E.FINGERPRINT)
    model = oracle.StoreModel(16, 12)
    n = 300
    cids, _ = E.gen_stream_ids(n, 0.4)
    off, nh = E.gen_addr(42, cids, 16)
    pages = np.stack([E.gen_chunk_host(42, int(c), 65536) for c in cids])
    u, l = nh, off >> np.uint64(16)
    lens = eng.put(u, l, pages, ts=np.arange(n, dtype=np.uint64))
    for i in range(n):
        model.put(int(off[i]), int(nh[i]), 0, pages[i])
    assert eng.entries() == model.entries()
    recs = eng.read_records(u, l)
    for i in range(n):
        assert recs[i] == model.record_bytes(int(u[i]), int(l[i])), i
    # lens: -1 for a chunk superseded by a later one of the same device batch (max_batch=256),
    # else the compressed_length that was stored when the chunk was applied
    last = {}
    for i in range(n):
        last[(int(u[i]), int(l[i]))] = i
    for i in range(n):
        later_same_batch = [j for j in range(i + 1, (i // 256 + 1) * 256) if j < n and (u[j], l[j]) == (u[i], l[i])]
        if later_same_batch:
            assert lens[i] == -1
        else:
            assert lens[i] == len(oracle.lz4_encode(pages[i], 12))
    fps, ok = eng.read_fingerprints(u, l)
    assert ok.all()
    for i in range(0, n, 17):
        assert (int(fps[i, 0]), int(fps[i, 1])) == oracle.fingerprint128(pages[last[(int(u[i]), int(l[i]))]])
    out, status = eng.get(u, l)
    assert (status == E.HIT).all() and all((out[i] == pages[last[(int(u[i]), int(l[i]))]]).all() for i in range(n))
    eng.close()


def test_store_semantics_vs_model(E, gpu, oracle):
    """Random put / get / unset batches against the store model: hit/miss, bad-entry, overwrite,
    entry count; 4 KiB pages so the oracle finishes in seconds."""
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=8192, arena_bytes=64 << 20, max_batch=128)
    model = oracle.StoreModel(pshift, 12)
    w = datagen.words(77, 4000)
    universe = [(int(w[i] % np.uint64(5)) + 1, int(w[i + 1] % np.uint64(300))) for i in range(0, 600, 2)]
    step = 0
    for rnd in range(12):
        k = 40 + rnd * 13
        pick = [universe[int(x % np.uint64(len(universe)))] for x in datagen.words(1000 + rnd, k)]
        u = np.array([p[0] for p in pick], dtype=np.uint64)
        l = np.array([p[1] for p in pick], dtype=np.uint64)
        if rnd % 3 != 2:
            pages = np.stack([datagen.make_page("RTZMPA"[(step + i) % 6], bs, step + i) for i in range(k)])
            eng.put(u, l, pages)
            for i in range(k):
                model.put(int(l[i]) << pshift, int(u[i]), 0, pages[i])
            step += k
        else:
            eng.unset(u[: k // 3], l[: k // 3])
            for i in range(k // 3):
                model.unset(int(u[i]), int(l[i]))
        assert eng.entries() == model.entries()
        q = [universe[int(x % np.uint64(len(universe)))] for x in datagen.words(2000 + rnd, 150)]
        qu = np.array([p[0] for p in q], dtype=np.uint64)
        ql = np.array([p[1] for p in q], dtype=np.uint64)
        out, status = eng.get(qu, ql)
        for i in range(len(q)):
            exp = model.get(int(ql[i]) << pshift, int(qu[i]), 0)
            assert (status[i] == E.HIT) == (exp is not None), (rnd, i)
            if exp is not None:
                assert out[i].tobytes() == exp
    st = eng.stats()
    assert st["dropped_puts"] == 0 and st["entries"] == model.entries()
    eng.close()


def test_raw_mode_and_other_page_sizes(E, gpu, oracle, tmp_path):
    for pshift, accel in ((12, 0), (13, 12), (15, 12), (17, 12), (16, 0),
                          *((ps, a) for ps in (6, 8, 10, 11, 18, 19, 20) for a in (12, 0))):
        cm = E.Cachemap(str(tmp_path), 2048, accel, pshift)
        bs = 1 << pshift
        n = 40
        pages = np.stack([datagen.make_page("RTZM"[i % 4], bs, 5 * pshift + i) for i in range(n)])
        off = (np.arange(n, dtype=np.uint64) * np.uint64(3)) << np.uint64(pshift)
        nh = np.full(n, 0xABCDEF, dtype=np.uint64)
        gen = np.zeros(n, dtype=np.uint32)
        cm.put_batch(off, nh, gen, pages)
        out, hit = cm.get_batch(off, nh, gen)
        assert hit.all() and (out == pages).all(), (pshift, accel)
        _, miss = cm.get_batch(off + np.uint64(bs), nh, gen)
        assert not miss.any()
        eng = E.Engine.__new__(E.Engine); eng.h = cm.engine_handle(); eng.bsize = bs
        recs = eng.read_records(nh, off >> np.uint64(pshift))
        model = oracle.StoreModel(pshift, accel)
        for i in range(n):
            model.put(int(off[i]), int(nh[i]), 0, pages[i])
            assert recs[i] == model.record_bytes(int(nh[i]), int(off[i]) >> pshift), (pshift, accel, i)
        eng.h = None
        assert cm.counters() == (2 * n, n)
        cm.free()


def test_concurrent_callers_are_combined(E, gpu, tmp_path):
    """libfuse runs edgefs_read/write on many threads (edgefs.c:78,2194): concurrent single-page
    calls must be safe and see their own writes."""
    cm = E.Cachemap(str(tmp_path), 4096, 12, 16)
    errs = []

    def worker(t):
        try:
            for i in range(12):
                page = datagen.make_page("RTZM"[(t + i) % 4], 65536, 100 * t + i)
                off = (t * 64 + i) << 16
                cm.put(off, 0x1000 + t, 0, page)
                back = cm.get(off, 0x1000 + t, 0)
                assert back == page.tobytes(), (t, i)
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs
    assert cm.counters() == (96, 96)
    cm.free()


def test_async_put_queue(E, gpu, tmp_path):
    cm = E.Cachemap(str(tmp_path), 4096, 12, 15)          # cachemap_test.c shape: 32 KiB pages
    pages = [datagen.make_page("TZ"[i % 2], 32768, i) for i in range(200)]
    for i, p in enumerate(pages):
        cm.put(i * 4096 * 8, 5 * i + 1, i, p, async_=True)
    cm_h = cm.h
    cm.free()                                             # drains the queue (cachemap.c:218-232)
    assert cm_h
    cm = E.Cachemap(str(tmp_path), 4096, 12, 15)
    for i, p in enumerate(pages[:50]):
        cm.put(i * 4096 * 8, 5 * i + 1, i, p, async_=True)
    import time
    deadline = time.time() + 20
    got = 0
    while time.time() < deadline:
        got = sum(cm.get(i * 4096 * 8, 5 * i + 1, i) == pages[i].tobytes() for i in range(50))
        if got == 50:
            break
        time.sleep(0.05)
    assert got == 50
    cm.free()


def test_eviction_keeps_capacity(E, gpu, tmp_path):
    """Policy equivalence only (SURVEY.md §8f-2): entries never exceed capacity, recent puts
    survive more often than old ones."""
    cm = E.Cachemap(str(tmp_path), 1024, 12, 12)
    bs = 4096
    total = 3000
    pages = np.stack([datagen.make_page("T", bs, i) for i in range(total)])
    nh = np.full(total, 9, dtype=np.uint64)
    gen = np.zeros(total, dtype=np.uint32)
    off = np.arange(total, dtype=np.uint64) << np.uint64(12)
    for at in range(0, total, 100):
        cm.put_batch(off[at:at + 100], nh[at:at + 100], gen[at:at + 100], pages[at:at + 100])
        import time
        time.sleep(0.005)                                 # CLOCK_REALTIME_COARSE granularity
    entries = E.lib().filemap_entries(_pages_ptr(cm))
    assert entries <= 1024
    _, hit = cm.get_batch(off, nh, gen)
    assert hit.sum() == entries
    assert hit[-500:].mean() > hit[:500].mean()
    cm.free()


def test_remote_index_import_records(E, gpu, oracle):
    """Multi-GPU index replica on one GPU: records written "elsewhere" are imported; per key the
    highest stream position wins whatever the arrival order (SURVEY.md 8e ordering caveat)."""
    from edge_fuse_b200 import sharding
    eng = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=32 << 20, max_batch=64)
    n = 100
    pages = np.stack([datagen.make_page("T", 4096, i) for i in range(n)])
    u = np.full(n, 5, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    eng.set_stream_order(1000, 2)                     # this rank owns positions 1000, 1002, ...
    eng.put(u, l, pages)
    assert eng.entries() == n
    # rank 1 wrote keys 0..49 later (odd positions above ours) and keys 50..59 earlier; key 200 is new.
    ru = np.full(61, 5, dtype=np.uint64)
    rl = np.concatenate([np.arange(60), [200]]).astype(np.uint64)
    rseq = np.concatenate([1001 + 2 * np.arange(50) + 2 * 200, 3 + np.arange(10), [7]]).astype(np.uint64)
    # duplicates inside one import: key 0 appears twice, the larger sequence must win
    ru = np.append(ru, np.uint64(5)); rl = np.append(rl, np.uint64(0)); rseq = np.append(rseq, np.uint64(5000))
    # rows 0..60 come from rank 1, the last from rank 3; no location (offset 0, length 0): only peer
    # reads, which this test does not make, would use one
    lens = np.zeros(len(ru), dtype=np.int64)
    rows = np.concatenate([sharding.pack_records(ru[:-1], rl[:-1], rseq[:-1], 1, lens[:-1]),
                           sharding.pack_records(ru[-1:], rl[-1:], rseq[-1:], 3, lens[-1:])])
    perm = np.argsort(datagen.words(9, len(ru)))      # arrival order must not matter
    rows = rows[perm]
    d_rows = eng.dev_alloc(rows.nbytes)
    eng.h2d(d_rows, rows)
    eng.import_records_dev(len(rows), d_rows, 0)
    eng.sync()
    eng.dev_free(d_rows)
    status, own = eng.locate(u, l)
    assert (status[:50] == E.REMOTE).all() and (status[50:] == E.HIT).all()
    assert own[0] == 3 and (own[1:50] == 1).all()
    st = eng.stats()
    assert st["entries"] == 50 and st["remote_entries"] == 51
    s2, o2 = eng.locate(np.array([5], dtype=np.uint64), np.array([200], dtype=np.uint64))
    assert s2[0] == E.REMOTE and o2[0] == 1
    out, gstat = eng.get(u, l)
    assert (gstat[:50] == E.REMOTE).all() and (gstat[50:] == E.HIT).all() and (out[50:] == pages[50:]).all()
    # a later local put takes the key back
    eng.set_stream_order(10_000, 2)
    eng.put(u[:5], l[:5], pages[:5])
    status, _ = eng.locate(u[:6], l[:6])
    assert (status[:5] == E.HIT).all() and status[5] == E.REMOTE
    assert eng.stats()["remote_entries"] == 46 and eng.entries() == 55
    eng.close()


def test_c_caller_links_like_edgefs(E, gpu, tmp_path):
    """A plain C program against include/cachemap.h and -lcachemap (the way edgefs links,
    Makefile:20,28): async inserts, read-back with byte checks, counters, the request-range calls
    with the glue header, checkpoint, free, and a second cachemap on the same directory."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "drop_in_test"
    lib_dir = os.path.dirname(E.library_path())
    subprocess.run(["gcc", "-std=c99", "-D_DEFAULT_SOURCE", "-O2", "-I", os.path.join(root, "include"),
                    os.path.join(root, "tests", "c", "drop_in_test.c"), "-L", lib_dir, "-lcachemap",
                    f"-Wl,-rpath,{lib_dir}", "-o", str(exe)], check=True)
    env = dict(os.environ, CMB200_ARENA_MB="512", CMB200_MAX_BATCH="512")
    for pshift, n in ((15, 300), (16, 200), (12, 500)):
        store = tmp_path / f"store{pshift}"
        store.mkdir()
        out = subprocess.run([str(exe), str(store), str(pshift), str(n)], capture_output=True, text=True, env=env,
                             timeout=200)
        assert out.returncode == 0, (pshift, out.returncode, out.stdout, out.stderr)
        assert "drop_in_test ok" in out.stdout and "ratio:" in out.stdout


def test_write_behind_ring_wraps_and_keeps_read_your_writes(E, gpu, tmp_path):
    """Single-page puts go through a page-locked write-behind ring.  With a ring of only 64 pages
    and 8 writer threads the ring wraps and back-pressures many times; every get that follows a
    put (same thread) must return that put's bytes, rewrites of one address must resolve to the
    last one, and nothing may be lost when the map is freed and the counters read."""
    import subprocess
    import sys
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import numpy as np, datagen, edge_fuse_b200 as E
cm = E.Cachemap(sys.argv[1], 8192, 12, 14)          # 16 KiB pages
bs = cm.bsize
errs = []
def worker(t):
    try:
        for i in range(300):
            page = datagen.make_page("RTZMPA"[(t + i) % 6], bs, 1000 * t + i)
            off = ((t * 40 + i % 40)) << 14             # 40 addresses per thread, rewritten ~7 times
            cm.put(off, 0xABC0 + t, 0, page)
            if i % 3 == 0:
                back = cm.get(off, 0xABC0 + t, 0)
                assert back == page.tobytes(), (t, i)
    except Exception as e:
        errs.append(repr(e))
th = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
[x.start() for x in th]; [x.join() for x in th]
assert not errs, errs[:3]
for t in range(8):                                     # final contents: the last write of each address
    for a in range(40):
        i = max(j for j in range(300) if j % 40 == a)
        want = datagen.make_page("RTZMPA"[(t + i) % 6], bs, 1000 * t + i).tobytes()
        assert cm.get((t * 40 + a) << 14, 0xABC0 + t, 0) == want, (t, a)
assert E.lib().filemap_entries(__import__("ctypes").cast(cm.h, __import__("ctypes").POINTER(__import__("ctypes").c_void_p))[0]) == 320
rq, ht = cm.counters()
assert rq == ht == 8 * 100 + 320, (rq, ht)
cm.free()
print("write-behind ok")
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CMB200_WB_SLOTS="64", CMB200_ARENA_MB="256", CMB200_MAX_BATCH="256")
    out = subprocess.run([sys.executable, "-c", code, str(tmp_path)], cwd=root, env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "write-behind ok" in out.stdout, out.stdout + out.stderr


def test_direct_arena_segments(gpu):
    """Large arenas take the direct path: blocks are encoded straight into per-warp arena segments
    (kernels.cu commit_direct) instead of passing through the stage buffer.  CMB200_SEG_KB forces
    small segments so that they roll over many times; records, lengths, rewrites in place and
    read-back must be what the staged path gives."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import sys, os
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
from oracle import ef_oracle as O
n = 3000
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=2 << 30, max_batch=1024, flags=E.FINGERPRINT)
u = np.full(n, 9, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
used = []
for rnd in range(3):                       # round 0 allocates, round 1 rewrites the same content, round 2 other content
    pages = np.stack([E.gen_chunk_host(7 + (rnd == 2), c, 65536) for c in range(n)])
    lens = eng.put(u, l, pages)
    st = eng.stats(); used.append((st["arena_used"], st["arena_garbage"]))
    out, status = eng.get(u, l)
    assert (status == E.HIT).all() and (out == pages).all(), rnd
    recs = eng.read_records(u, l)
    for k in list(range(0, n, 83)) + [n - 1]:
        blk = O.lz4_encode(pages[k], 12)
        assert recs[k][24:] == blk and recs[k][:16] == np.array([9, k], dtype=np.uint64).tobytes(), (rnd, k)
        assert int(lens[k]) == len(blk) == int.from_bytes(recs[k][16:20], "little"), (rnd, k)
    fps, ok = eng.read_fingerprints(u, l)
    assert ok.all() and (int(fps[5, 0]), int(fps[5, 1])) == O.fingerprint128(pages[5])
st = eng.stats()
assert st["entries"] == n and st["dropped_puts"] == 0 and st["arena_used"] <= (2 << 30), st
print("direct ok", used)
'''
    env = dict(os.environ, CMB200_SEG_KB="320")
    out = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "direct ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("seg_kb", ["0", "1"])       # stage rows / arena segments of one worst-case record
@pytest.mark.parametrize("pshift", [18, 19, 20])
def test_incompressible_large_pages_are_stored_raw(E, gpu, oracle, tmp_path, monkeypatch, pshift, seg_kb):
    """Above 128 KiB an incompressible page's block is longer than the bsize + 1024 bytes filemap_set
    gives LZ4_compress_fast; the page is stored raw (compressed_length 0, DESIGN.md f1) and the block,
    written first, stays inside its stage row or arena segment.  Random pages alternate with
    compressible ones so that neighbouring warps encode at the same time."""
    monkeypatch.setenv("CMB200_SEG_KB", seg_kb)
    monkeypatch.setenv("CMB200_PERSIST", "0")
    bs, n, nh = 1 << pshift, {18: 256, 19: 160, 20: 128}[pshift], 0xB16
    pages = np.stack([datagen.make_page("R" if i % 2 == 0 else "TX"[i // 2 % 2], bs, 31 * pshift + i) for i in range(n)])
    u = np.full(n, nh, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    model = oracle.StoreModel(pshift, 12)
    for i in range(n):
        model.put(i << pshift, nh, 0, pages[i])
    exp = [model.record_bytes(nh, i) for i in range(n)]
    exp_lens = [int.from_bytes(r[16:20], "little") for r in exp]
    assert exp_lens.count(0) >= n // 4 and min(exp_lens[1::2]) > 0
    row = 24 + max(bs + 1024, bs + bs // 255 + 16) + 16
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=3 * n * row + (64 << 20), max_batch=256)
    path = str(tmp_path / "large.snap")
    eng = E.Engine(**geo)                      # one engine at a time: the stage alone is ~17 GB at 2^20
    try:
        lens = eng.put(u, l, pages)
        assert lens.tolist() == exp_lens
        assert eng.read_records(u, l) == exp
        out, st = eng.get(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
        assert eng.stats()["dropped_puts"] == 0
        assert eng.save(path) == n
    finally:
        eng.close()
    eng = E.Engine(**geo)
    try:
        assert eng.load(path) == n
        assert eng.read_records(u, l) == exp
        out, st = eng.get(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
    finally:
        eng.close()
    cm = E.Cachemap(str(tmp_path), 1024, 12, pshift)
    off = l << np.uint64(pshift)
    gen = np.zeros(n, dtype=np.uint32)
    cm.put_batch(off, u, gen, pages)
    out, hit = cm.get_batch(off, u, gen)
    assert hit.all() and (out == pages).all()
    view = E.Engine.__new__(E.Engine); view.h = cm.engine_handle(); view.bsize = bs
    assert view.read_records(u, l) == exp
    assert view.stats()["dropped_puts"] == 0
    view.h = None
    cm.free()


@pytest.mark.gpu
@pytest.mark.parametrize("pshift", [12, 16])
def test_request_ranges_follow_the_fuse_loops(E, gpu, oracle, tmp_path, pshift):
    """cachemap_read_range / _write_range against the page loops of edgefs_read / edgefs_write
    (edgefs.c:1150-1195, 1216-1228) replayed on the store model: same bytes, same hit/miss answer
    per request, same requests / hits counters (pages after the first miss are never asked for)."""
    import datagen
    page = 1 << pshift
    cm = E.Cachemap(str(tmp_path), 4096, 12, pshift)
    model = oracle.StoreModel(pshift, 12)
    rng = np.random.default_rng(pshift)
    nhids = [oracle.build_nhid(b"obj%d" % i, b"/bk1") for i in range(3)]
    span = 64                                           # pages per object that the trace touches
    for step in range(400):
        nh = nhids[int(rng.integers(0, 3))]
        first = int(rng.integers(0, span))
        npages = int(rng.integers(1, min(32, 131072 // page) + 1))      # max_write 131072 (edgefs.c:1366)
        off, size = first * page, npages * page
        kind = rng.random()
        if kind < 0.08:                                 # unaligned requests bypass the cache
            off += int(rng.integers(1, page))
        elif kind < 0.12:
            size -= int(rng.integers(1, page))
        elif kind < 0.15:
            off = ((1 << 44) - 1) * page if pshift == 16 else off     # last valid page, then invalid ones
        if rng.random() < 0.45:
            data = b"".join(datagen.make_page("RTZMPAXS"[int(rng.integers(0, 8))], page, step * 40 + j).tobytes()
                            for j in range((size + page - 1) // page))[:size]
            cm.write_range(nh, 0, off, data)
            model.write_range(nh, 0, off, data)
        else:
            got = cm.read_range(nh, 0, off, size)
            want = model.read_range(nh, 0, off, size)
            assert got == want, (step, off, size)
        assert cm.counters() == (model.requests, model.hits), step
    assert cm.read_range(nhids[0], 0, 0, 0) == b""      # empty request: the loop body never runs
    cm.free()


def test_async_put_batches_overlap_and_stay_ordered(E, gpu, oracle):
    """cmb200_put_batch_async returns once the host arrays have crossed: the same host buffer is
    refilled for the next batch straight away, the stored lengths arrive behind the ticket, and
    later calls (rewrites of the same keys, gets) are ordered after the pending encode."""
    n, rounds = 1500, 5
    eng = E.Engine(pshift=16, accel=12, capacity=16384, arena_bytes=1 << 30, max_batch=512, flags=E.FINGERPRINT)
    ct = np.ctypeslib.ctypes
    hp = E.lib().cmb200_host_alloc(n * 65536)
    pages = np.ctypeslib.as_array((ct.c_uint8 * (n * 65536)).from_address(hp)).reshape(n, 65536)
    lens_pin = []
    for _ in range(2):
        p = E.lib().cmb200_host_alloc(n * 4)
        lens_pin.append((p, np.ctypeslib.as_array((ct.c_int32 * n).from_address(p))))
    src = [np.stack([E.gen_chunk_host(100 + r, c, 65536) for c in range(n)]) for r in range(rounds)]
    sample = list(range(0, n, 61))
    u = np.full(n, 5, dtype=np.uint64)
    tickets = []

    def check_lens(r):
        eng.wait(tickets[r])
        got = lens_pin[r & 1][1]
        assert (got > 0).all(), r
        for k in sample:
            assert int(got[k]) == len(oracle.lz4_encode(src[r][k], 12)), (r, k)

    for r in range(rounds):
        l = np.arange(n, dtype=np.uint64) + np.uint64((r % 2) * (n // 2))      # half the keys get rewritten
        if r >= 2:
            check_lens(r - 2)                                                   # frees lens_pin[r & 1]
        pages[:] = src[r]                                                       # host buffer reused at once
        tickets.append(eng.put_async(u, l, pages, lens=lens_pin[r & 1][0]))
    check_lens(rounds - 2)
    check_lens(rounds - 1)
    newest = {}
    for r in range(rounds):
        for k in range(n):
            newest[k + (r % 2) * (n // 2)] = (r, k)
    keys = np.array(sorted(newest), dtype=np.uint64)
    out, status = eng.get(np.full(len(keys), 5, dtype=np.uint64), keys)
    assert (status == E.HIT).all()
    for i, key in enumerate(keys):
        r, k = newest[int(key)]
        assert (out[i] == src[r][k]).all(), (int(key), r, k)
    assert eng.entries() == len(keys)
    eng.wait(0)
    eng.wait(tickets[0])                                                        # stale tickets return at once
    st = eng.stats()
    assert st["put_chunks"] == n * rounds and st["dropped_puts"] == 0
    for p in [hp] + [x[0] for x in lens_pin]:
        E.lib().cmb200_host_free(p)
    eng.close()


def test_cache_directory_survives_a_restart(E, gpu, oracle, tmp_path):
    """The reference's store is its LMDB files, so a cache directory keeps its pages across
    restarts (filemap.c:57,71-72).  Here cachemap_free / cachemap_checkpoint write
    <dir>/cachemap_b200.snap and the next cachemap_create on that directory reads it back:
    same hits, same pages, same record bytes, same entry count; counters start from zero."""
    d = tmp_path / "cache"
    d.mkdir()
    n = 700
    cm = E.Cachemap(str(d), 4096, 12, 16)
    model = oracle.StoreModel(16, 12)
    pages = [datagen.make_page("RTZMPAXS"[i % 8], 65536, 900 + i) for i in range(n)]
    for i in range(n):
        off, nh = (i % 500) << 16, 77 + (i % 3)          # some addresses are rewritten
        cm.put(off, nh, 0, pages[i])
        model.put(off, nh, 0, pages[i])
    assert cm.checkpoint() == 0 and (d / "cachemap_b200.snap").exists()
    cm.put(499 << 16, 77, 5, pages[0])                   # after the checkpoint: saved again by free
    model.put(499 << 16, 77, 5, pages[0])
    cm.free()

    cm2 = E.Cachemap(str(d), 4096, 12, 16)
    assert cm2.counters() == (0, 0)
    for i in range(0, 500, 7):
        for nh in (77, 78, 79):
            got, want = cm2.get(i << 16, nh, 0), model.get(i << 16, nh, 0)
            assert (got is None) == (want is None) and (got is None or got == bytes(want)), (i, nh)
    assert cm2.get(499 << 16, 77, 5) == bytes(pages[0])
    assert E.lib().cmb200_entries(cm2.engine_handle()) == model.entries()
    cm2.free()

    # a directory written with another page size is ignored (message on stderr), not misread
    cm3 = E.Cachemap(str(d), 4096, 12, 12)
    assert cm3.get(0, 77, 0) is None
    cm3.put(0, 77, 0, pages[1][:4096])
    assert cm3.get(0, 77, 0) == bytes(pages[1][:4096])
    cm3.free()


def test_engine_snapshot_roundtrip_any_geometry(E, gpu, oracle, tmp_path):
    """cmb200_save / cmb200_load at the engine level: record bytes, timestamps and fingerprints come
    back identical in an engine with a different capacity and arena; raw records (accel 0) too."""
    n = 1200
    pages = np.stack([E.gen_chunk_host(11, c, 65536) for c in range(n)])
    u = np.full(n, 3, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    ts = np.arange(n, dtype=np.uint64) + np.uint64(1000)
    for accel in (12, 0):
        a = E.Engine(pshift=16, accel=accel, capacity=4096, arena_bytes=256 << 20, max_batch=512, flags=E.FINGERPRINT)
        a.put(u, l, pages, ts=ts)
        a.unset(u[:100], l[:100])                                     # deleted records are not saved
        path = str(tmp_path / f"snap{accel}")
        assert a.save(path) == n - 100
        b = E.Engine(pshift=16, accel=accel, capacity=65536, arena_bytes=1 << 30, max_batch=256, flags=E.FINGERPRINT)
        assert b.load(path) == n - 100 and b.entries() == n - 100
        ra, rb = a.read_records(u, l), b.read_records(u, l)
        assert ra == rb and ra[0] is None and ra[100] is not None
        fa, oka = a.read_fingerprints(u, l)
        fb, okb = b.read_fingerprints(u, l)
        assert (oka == okb).all() and (fa[oka != 0] == fb[okb != 0]).all()
        out, st = b.get(u, l)
        assert (st[:100] == E.MISS).all() and (st[100:] == E.HIT).all() and (out[100:] == pages[100:]).all()
        r = np.arange(40, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        _, tsb, okb2 = b.sample(r)
        assert okb2.all() and ((tsb >= 1100) & (tsb < 1000 + n)).all()  # the LMDB attribute travels too
        a.close(); b.close()
    c = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=256)
    with pytest.raises(Exception):
        c.load(str(tmp_path / "snap12"))                               # other page size
    c.close()


def test_put_step_records_and_device_import(E, gpu, oracle):
    """cmb200_put_step packs the exchange records of a step on the device exactly as sharding.py
    packs them on the host, and cmb200_import_records_dev applies all-gathered records: own rows and
    rows that stored nothing are skipped, the newest stream position per key wins."""
    from edge_fuse_b200 import sharding
    n, world, rank = 512, 4, 1
    eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=128 << 20, max_batch=256, flags=E.FINGERPRINT)
    pages = np.stack([E.gen_chunk_host(3, c, 65536) for c in range(n)])
    d_pages = eng.dev_alloc(n * 65536)
    eng.h2d(d_pages, pages)
    d_rec = eng.dev_alloc(n * 32)
    u = np.full(n, 21, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    l[100] = l[40]                                                  # same key twice in the step: 40 is superseded
    valid = np.ones(n, dtype=np.uint8); valid[7] = 0                # rejected address
    base = 1000
    eng.set_stream_order(base + rank, world)
    hp = E.lib().cmb200_host_alloc(n * 65536)                      # page-locked copy for mode 2
    pinned = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint8 * (n * 65536)).from_address(hp)).reshape(n, 65536)
    pinned[:] = pages
    for on_dev, src in ((True, d_pages), (False, pages), (2, pinned)):
        tk = eng.put_step(u, l, src, valid=valid, on_dev=on_dev, rank=rank, records_dev=d_rec)
        eng.wait(tk); eng.sync()
        got = np.zeros((n, 4), dtype=np.int64)
        eng.d2h(got, d_rec)
        pos = sharding.shard_positions(rank, world, n, base)
        lens = np.array([len(oracle.lz4_encode(pages[i], 12)) for i in range(n)], dtype=np.int64)
        lens[7] = -1; lens[40] = -1
        want = sharding.pack_records(u, l, pos, rank, lens)
        assert (got[:, :3] == want[:, :3]).all(), on_dev
        for a, b in zip(sharding.unpack_records(got)[3:], sharding.unpack_records(want)[3:]):
            assert (a == b).all(), on_dev                            # owner rank, stored length (-1 = nothing stored)
        loc = sharding.unpack_locations(got).astype(np.uint64)       # where each record lies in this rank's arena
        stored = lens >= 0
        assert (loc[~stored] == 0).all() and (loc[stored] % 16 == 0).all()
        assert len(set(loc[stored].tolist())) == int(stored.sum()) and loc[stored].max() < eng.stats()["arena_used"]
        base += world * n
        eng.set_stream_order(base + rank, world)
    assert eng.entries() == n - 2
    # "all-gathered" rows: ours (ignored), another rank rewriting key 5 later (wins), another rank with
    # an older position for key 6 (loses), a row that stored nothing (ignored), a new remote key
    rows = np.concatenate([
        sharding.pack_records([21], [5], [base + 10], rank, [100]),
        sharding.pack_records([21], [5], [base + 50], 2, [200], rec_off=[4096]),
        sharding.pack_records([21], [6], [3], 3, [300]),
        sharding.pack_records([21], [9], [base + 60], 2, [-1]),
        sharding.pack_records([99], [1], [base + 70], 0, [400], rec_off=[1 << 20]),
    ])
    d_rows = eng.dev_alloc(rows.nbytes)
    eng.h2d(d_rows, rows)
    eng.import_records_dev(len(rows), d_rows, rank)
    eng.sync()
    status, owner = eng.locate(np.array([21, 21, 21, 99], dtype=np.uint64), np.array([5, 6, 9, 1], dtype=np.uint64))
    assert list(status) == [E.REMOTE, E.HIT, E.HIT, E.REMOTE] and owner[0] == 2 and owner[3] == 0
    st = eng.stats()
    assert st["entries"] == n - 3 and st["remote_entries"] == 2
    for p in (d_pages, d_rec, d_rows):
        eng.dev_free(p)
    eng.close()
    E.lib().cmb200_host_free(hp)


def test_import_gathered_host_and_device_tensors(E, gpu):
    """sharding.import_gathered takes an all-gathered record tensor on the host or on the device,
    imports the other ranks' rows that stored something before it returns, and returns their number."""
    import torch
    from edge_fuse_b200 import sharding
    rows = np.concatenate([
        sharding.pack_records([7, 7], [1, 2], [10, 11], 0, [100, 100]),          # this rank's own rows
        sharding.pack_records([7, 7], [3, 4], [12, 13], 1, [100, -1]),           # key 4 stored nothing
        sharding.pack_records([7], [5], [14], 2, [100], rec_off=[4096]),
    ])
    for gathered in (torch.from_numpy(rows), torch.from_numpy(rows).cuda()):
        eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
        assert sharding.import_gathered(eng, gathered[:2], 0) == 0
        assert sharding.import_gathered(eng, gathered, 0) == 2
        status, owner = eng.locate(np.full(5, 7, dtype=np.uint64), np.arange(1, 6, dtype=np.uint64))
        assert list(status) == [E.MISS, E.MISS, E.REMOTE, E.MISS, E.REMOTE], gathered.device
        assert owner[2] == 1 and owner[4] == 2 and eng.stats()["remote_entries"] == 2
        eng.close()


def test_device_pages_must_be_16_byte_aligned(E, gpu, oracle):
    """The encoder reads device pages with 16-byte loads, so put_batch_dev and put_step(on_dev=1)
    refuse a pointer that is only 4-byte aligned before anything is queued: no kernel is launched
    and the store is unchanged.  The same pages at a 16-byte aligned address store the reference's
    records."""
    n = 8
    eng = E.Engine(pshift=16, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.FINGERPRINT)
    pages = np.stack([E.gen_chunk_host(5, c, 65536) for c in range(n)])
    d_pages = eng.dev_alloc(n * 65536 + 256)
    d_rec = eng.dev_alloc(n * 32)
    u = np.full(n, 77, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    keys = ("entries", "put_chunks", "dropped_puts", "kernel_launches")
    before = eng.stats()
    eng.h2d(d_pages + 4, pages)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        eng.put(u, l, d_pages + 4, on_dev=True)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        eng.put_step(u, l, d_pages + 4, on_dev=True, records_dev=d_rec)
    eng.sync()
    after = eng.stats()
    assert {k: after[k] for k in keys} == {k: before[k] for k in keys}
    eng.h2d(d_pages + 16, pages)
    eng.put(u, l, d_pages + 16, on_dev=True)
    eng.wait(eng.put_step(u, l + np.uint64(n), d_pages + 16, on_dev=True, records_dev=d_rec))
    assert eng.entries() == 2 * n
    recs = eng.read_records(np.concatenate([u, u]), np.concatenate([l, l + np.uint64(n)]))
    for i in range(2 * n):
        blk = oracle.lz4_encode(pages[i % n], 12)
        assert recs[i] == oracle.record_prefix(77, i, len(blk)) + blk, i
    for p in (d_pages, d_rec):
        eng.dev_free(p)
    eng.close()


def test_arena_compaction_reclaims_deleted_and_outgrown_records(E, gpu, oracle):
    """cmb200_compact slides the live records down: arena_used falls to the live bytes, garbage to
    zero, and every record, timestamp and fingerprint is what it was (staged and in-place paths)."""
    import subprocess
    import sys
    code = r'''
import sys, os
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n = 1500
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=int(os.environ["ARENA"]), max_batch=512, flags=E.FINGERPRINT)
u = np.full(n, 4, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
small = np.stack([E.gen_chunk_host(1, 8 * c + 2, 65536) for c in range(n)])       # Z class: tiny records
big = np.stack([E.gen_chunk_host(1, 8 * c + 0, 65536) for c in range(n)])         # R class: outgrow them
eng.put(u, l, small, ts=np.arange(n, dtype=np.uint64))
eng.put(u[::2], l[::2], np.ascontiguousarray(big[::2]), ts=np.arange(n, dtype=np.uint64)[::2] + 5000)   # every other key outgrows its record
eng.unset(u[1::4], l[1::4])                                                        # and a quarter is deleted
before = eng.stats()
recs = eng.read_records(u, l); fps, ok = eng.read_fingerprints(u, l)
got = eng.compact()
after = eng.stats()
assert after["entries"] == before["entries"] and after["arena_garbage"] == 0 and got > 0
live = sum((len(r) + 15) & ~15 for r in recs if r is not None)
assert after["arena_used"] == live and before["arena_used"] - after["arena_used"] == got, (after, live, got)
assert eng.read_records(u, l) == recs
fps2, ok2 = eng.read_fingerprints(u, l)
assert (ok == ok2).all() and (fps[ok != 0] == fps2[ok2 != 0]).all()
out, st = eng.get(u, l)
want = small.copy(); want[::2] = big[::2]
hit = st == E.HIT
assert (hit == np.array([r is not None for r in recs])).all() and (out[hit] == want[hit]).all()
# the store keeps working: new puts land after the compacted records
eng.put(u[1::4], l[1::4], np.ascontiguousarray(big[1::4]))
out, st = eng.get(u, l)
assert (st == E.HIT).all() and (out[1::4] == big[1::4]).all() and eng.stats()["dropped_puts"] == 0
assert eng.compact() >= 0                                                          # idempotent on a tidy arena
print("compact ok", before["arena_used"], after["arena_used"])
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for arena, seg in ((256 << 20, "0"), (1 << 30, "320")):                    # staged path / in-place path
        env = dict(os.environ, ARENA=str(arena), CMB200_SEG_KB=seg)
        out = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and "compact ok" in out.stdout, out.stdout + out.stderr


def test_cache_outlives_many_times_its_arena(E, gpu, tmp_path, monkeypatch):
    """A cache that runs for a long time writes many times its arena.  With eviction holding the
    entry count at `capacity` and compaction reclaiming what eviction frees, no put is ever
    dropped and the newest pages are always readable (the reference's LMDB reuses freed pages)."""
    monkeypatch.setenv("CMB200_ARENA_MB", "96")
    monkeypatch.setenv("CMB200_SEG_KB", "0")
    cap = 1024
    cm = E.Cachemap(str(tmp_path), cap, 12, 16)
    pages = np.stack([E.gen_chunk_host(9, 8 * c, 65536) for c in range(256)])     # incompressible: 64 KiB records
    total = 6000                                                                    # ~375 MiB through a 96 MiB arena
    for base in range(0, total, 256):
        k = min(256, total - base)
        off = (np.arange(base, base + k, dtype=np.uint64)) << np.uint64(16)
        cm.put_batch(off, np.full(k, 3, dtype=np.uint64), np.zeros(k, dtype=np.uint32), pages[:k])
    import ctypes
    from edge_fuse_b200.binding import Stats
    eng_stats = Stats()
    assert E.lib().cmb200_get_stats(cm.engine_handle(), ctypes.byref(eng_stats)) == 0
    assert eng_stats.dropped_puts == 0 and eng_stats.entries <= cap
    # the pages of the last batch (put after the last eviction) are all there
    off = (np.arange(total - 100, total, dtype=np.uint64)) << np.uint64(16)
    out, hit = cm.get_batch(off, np.full(100, 3, dtype=np.uint64), np.zeros(100, dtype=np.uint32))
    assert hit.all() and (out == pages[(np.arange(total - 100, total) % 256)]).all()
    cm.free()


def test_snapshot_format_against_an_independent_writer_and_reader(E, gpu, oracle, tmp_path):
    """The snapshot file is a contract of its own: a file written by oracle/snapshot.py from the
    oracle's store model (records = the reference's LMDB values) loads into the engine and serves
    the model's pages, and a file written by the engine parses back to exactly the model's records."""
    from oracle import snapshot
    n = 400
    model = oracle.StoreModel(16, 12)
    pages = [datagen.make_page("RTZMPAXS"[i % 8], 65536, 7000 + i) for i in range(n)]
    addrs = []
    for i in range(n):
        off, nh = (i % 300) << 16, 40 + (i % 2)
        model.put(off, nh, 0, pages[i])
        addrs.append(oracle.addr_compose(off, nh, 0, 16))
    keys = sorted(set(addrs))
    recs = [(1000 + j, 0, 0, model.record_bytes(u, l)) for j, (u, l) in enumerate(keys)]
    path = str(tmp_path / "model.snap")
    snapshot.write_snapshot(path, 16, recs)
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=256 << 20, max_batch=256)
    assert eng.load(path) == len(keys) and eng.entries() == model.entries()
    u = np.array([k[0] for k in keys], dtype=np.uint64)
    l = np.array([k[1] for k in keys], dtype=np.uint64)
    assert eng.read_records(u, l) == [r[3] for r in recs]
    out, status = eng.get(u, l)
    assert (status == E.HIT).all()
    for j, (ku, kl) in enumerate(keys):
        want = model.get(int(kl) << 16, int(ku), 0)          # l = page number (genid 0), u = nhid
        assert want is not None and bytes(out[j]) == bytes(want), j
    # and back: what the engine writes is what the independent reader expects
    path2 = str(tmp_path / "engine.snap")
    assert eng.save(path2) == len(keys)
    pshift, flags, got = snapshot.read_snapshot(path2)
    assert pshift == 16 and flags == 0
    assert sorted(r[3] for r in got) == sorted(r[3] for r in recs)
    assert sorted(r[0] for r in got) == sorted(r[0] for r in recs)       # timestamps travel
    eng.close()


@pytest.mark.gpu
def test_full_arena_drops_puts_but_never_corrupts(E, gpu, oracle):
    """An arena that runs full with records of mixed sizes: a put that does not fit is dropped (a
    full LMDB map drops it, filemap.c:143-145,154-157) and every key that still HITs returns its
    own page byte for byte.  The bump pointer is never rolled back (it saturates until the arena is
    compacted), so no allocation can ever overlap a record that was stored."""
    import subprocess
    import sys
    code = r'''
import sys, os
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n = 2048
# arena: ~40 % of what the mixed batch needs -> many drops, small records keep fitting near the end
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=int(os.environ["ARENA"]), max_batch=512)
u = np.full(n, 11, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
# incompressible (66 KiB records) interleaved with zero pages (~300-byte records) and text pages
cids = np.array([8 * c + (0, 2, 1, 2)[c & 3] for c in range(n)], dtype=np.uint64)
pages = np.stack([E.gen_chunk_host(3, int(c), 65536) for c in cids])
for rep in range(3):                       # the later rounds run against an arena that is already full
    lens = eng.put(u, l, pages)
    out, st = eng.get(u, l)
    hit = st == E.HIT
    assert (out[hit] == pages[hit]).all(), "a HIT returned another page's bytes"
    assert ((st == E.HIT) | (st == E.MISS)).all()
    stats = eng.stats()
    assert stats["dropped_puts"] > 0 and stats["arena_used"] <= stats["arena_bytes"]
    assert stats["entries"] == int(hit.sum())
assert 0 < hit.sum() < n
print("full arena ok", int(hit.sum()), stats["dropped_puts"])
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for arena, seg in ((24 << 20, "0"), (40 << 20, "320")):                     # staged path / per-warp segments
        env = dict(os.environ, ARENA=str(arena), CMB200_SEG_KB=seg)
        out = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and "full arena ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_large_batches_at_capacity_stay_at_capacity(E, gpu, tmp_path, monkeypatch):
    """cachemap_put_batch with far more pages than the store's capacity, repeatedly: eviction runs
    before every slice of the batch (no fixed number of rounds), entries end within capacity, nothing
    is dropped, and the newest pages are the ones that survive."""
    monkeypatch.setenv("CMB200_ARENA_MB", "160")
    cap = 2048
    cm = E.Cachemap(str(tmp_path), cap, 12, 12)
    bs = 4096
    n = 20000                                              # ~10 x capacity in ONE call
    pages = np.stack([datagen.make_page("TRZM"[i & 3], bs, i) for i in range(512)])
    idx = np.arange(n) % 512
    nh = np.full(n, 21, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    for rnd in range(2):
        off = (np.arange(rnd * n, (rnd + 1) * n, dtype=np.uint64)) << np.uint64(12)
        cm.put_batch(off, nh, gen, np.ascontiguousarray(pages[idx]))
        entries = E.lib().filemap_entries(_pages_ptr(cm))
        assert entries <= cap + cap // 4, entries        # one slice (capacity / 4) of slack at most
        assert entries >= cap // 2
    import ctypes
    from edge_fuse_b200.binding import Stats
    st = Stats()
    assert E.lib().cmb200_get_stats(cm.engine_handle(), ctypes.byref(st)) == 0
    assert st.dropped_puts == 0
    out, hit = cm.get_batch(off[-256:], nh[-256:], gen[-256:])
    assert hit.mean() > 0.9 and (out[hit != 0] == pages[idx[-256:]][hit != 0]).all()
    cm.free()


@pytest.mark.gpu
def test_sampling_a_nearly_empty_table_and_corrupt_snapshots(E, gpu, oracle, tmp_path):
    """(1) filemap_get_rand's policy equivalent on a table with 3 live slots out of 2^20: the bounded
    walk gives up and the cooperative scan finds them (k_sample / k_sample_scan).
    (2) cmb200_load refuses records whose compressed_length disagrees with their length, and records
    whose length is below 24 or above 24 + bsize + 1024."""
    eng = E.Engine(pshift=12, accel=12, capacity=1 << 18, arena_bytes=16 << 20, max_batch=256)
    assert eng.stats()["table_slots"] >= 1 << 20
    r = datagen.words(77, 64)
    _, _, ok = eng.sample(r)
    assert (np.asarray(ok) == 0).all()                    # empty store: no victim
    pages = np.stack([datagen.make_page("T", 4096, i) for i in range(3)])
    u = np.full(3, 8, dtype=np.uint64); l = np.array([5, 6, 7], dtype=np.uint64)
    eng.put(u, l, pages, ts=np.array([10, 20, 30], dtype=np.uint64))
    addr, ts, ok = eng.sample(r)
    assert (np.asarray(ok) == 1).all()
    got = {(int(a[0]), int(a[1]), int(t)) for a, t in zip(np.asarray(addr).reshape(-1, 2), ts)}
    assert got <= {(8, 5, 10), (8, 6, 20), (8, 7, 30)} and len(got) >= 2
    # ---- corrupt snapshot ----
    snap = str(tmp_path / "s.snap")
    assert eng.save(snap) == 3
    raw = bytearray(open(snap, "rb").read())
    # record 0: header 64 B, record header 32 B {ts, fp, len, 0}, then data_prefix {u, l, compressed_length, pad}
    len_at, clen_at = 64 + 24, 64 + 32 + 16
    good = int.from_bytes(raw[clen_at:clen_at + 4], "little", signed=True)
    assert 0 < good < 4096 + 1024
    cases = [(clen_at, bad) for bad in (-5, good + 7, 0x7fffffff)] + [(len_at, 23), (len_at, 24 + 4096 + 1025)]
    for at, bad in cases:
        broken = bytearray(raw)
        broken[at:at + 4] = int(bad).to_bytes(4, "little", signed=True)
        p = str(tmp_path / f"bad{at}_{bad & 0xffff}.snap")
        open(p, "wb").write(broken)
        e2 = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=16 << 20, max_batch=256)
        with pytest.raises(RuntimeError):
            e2.load(p)
        out, st = e2.get(u, l)                             # the engine is still usable and holds nothing wrong
        assert ((st == E.MISS) | ((st == E.HIT) & (out == pages).all(axis=1))).all()
        e2.close()
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pshift", [12, 16])
def test_fused_small_get_matches_the_batch_get(E, gpu, oracle, pshift):
    """cmb200_get_small (lookup + TMA-staged record + shared-memory decode in one kernel) answers
    exactly like cmb200_get_batch: pages, HIT / MISS / BAD_ENTRY, raw pages, every content class."""
    bs = 1 << pshift
    kinds = "RTZMPAX"
    n = 70
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], bs, 100 + i) for i in range(n)])
    for accel in (12, 0):                                      # compressed records / raw pages (comp_accel == 0)
        eng = E.Engine(pshift=pshift, accel=accel, capacity=4096, arena_bytes=64 << 20, max_batch=64)
        u = np.full(n, 31, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        qu = np.concatenate([u, np.full(5, 32, dtype=np.uint64)])
        ql = np.concatenate([l, np.arange(5, dtype=np.uint64)])        # 5 misses
        out_b, st_b = eng.get(qu, ql)
        out_s, st_s = eng.get_small(qu, ql)
        assert (st_s == st_b).all() and (st_s[:n] == E.HIT).all() and (st_s[n:] == E.MISS).all()
        assert (out_s[:n] == pages).all() and (out_b[:n] == pages).all()
        # a rewrite is served from its new record, an unset key misses
        eng.put(u[:10], l[:10], pages[10:20])
        eng.unset(u[20:25], l[20:25])
        out_s, st_s = eng.get_small(u[:30], l[:30])
        assert (out_s[:10] == pages[10:20]).all() and (st_s[20:25] == E.MISS).all() and (st_s[:20] == E.HIT).all()
        assert (st_s[25:30] == E.HIT).all() and (out_s[25:30] == pages[25:30]).all()
        s = eng.stats()
        assert s["get_requests"] >= 2 * (n + 5) and s["dropped_puts"] == 0
        eng.close()


@pytest.mark.gpu
def test_small_gets_overlap_puts_without_torn_pages(E, gpu, tmp_path):
    """Readers on the get stream while a writer keeps rewriting the same keys with pages of two
    different contents (different record sizes): every get returns one of the two pages in full —
    the reference's LMDB readers see a snapshot (filemap.c:223-231), never a half-written record."""
    import subprocess
    import sys
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 192, 65536
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=3 << 30, max_batch=256)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])       # text-like: ~63 KiB records
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])       # half repeats: ~31 KiB records
u = np.full(n, 77, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
eng.put(u, l, A)
stop = threading.Event(); bad = []; gets = [0]
def reader():
    while not stop.is_set():
        out, st = eng.get_small(u, l)
        gets[0] += 1
        ok = (st == E.HIT) & ((out == A).all(axis=1) | (out == B).all(axis=1))
        if not ok.all():
            bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
            return
th = [threading.Thread(target=reader) for _ in range(2)]
[t.start() for t in th]
for rnd in range(40):
    eng.put(u, l, B if rnd % 2 == 0 else A)
stop.set(); [t.join() for t in th]
assert not bad, bad
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
print("no torn pages", gets[0], eng.stats()["arena_garbage"] > 0)
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_reference_exerciser_hit_ratios(E, gpu, tmp_path):
    """The reference's only exerciser (cachemap/cachemap_test.c: 32 768 x 32 KiB objects, capacity ==
    count, half re-put under new generation ids -> one eviction per put) run from one source
    (tests/c/exerciser.c) against this library and, linked against the reference's library, recorded
    in tests/golden/ref_exerciser.json: the hit ratio of every phase must agree within 2 points
    (eviction is random and wall-clock driven, so victims differ; the policy — oldest of three random
    records, cachemap.c:17-48 — must not)."""
    import re
    import subprocess
    import tempfile
    gold = json.load(open(os.path.join(GOLD, "ref_exerciser.json")))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "c", "exerciser.c")
    inc = os.path.join(root, "include")
    lib_dir = os.path.join(root, "edge_fuse_b200")
    ours = str(tmp_path / "exer_ours")
    subprocess.check_call(["gcc", "-O2", "-I", inc, src, "-o", ours, "-L", lib_dir, "-lcachemap", f"-Wl,-rpath,{lib_dir}", "-lpthread"])
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None

    def run(seed):
        with tempfile.TemporaryDirectory(dir=base) as d:
            env = dict(os.environ, CMB200_ARENA_MB="2048", CMB200_PERSIST="0")
            out = subprocess.run([ours, d, str(gold["objects"]), str(gold["pshift"]), str(seed)], capture_output=True,
                                 text=True, timeout=300, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        got = {m.group(1): int(m.group(2)) / int(m.group(3)) for m in re.finditer(r"phase (\w+) hits (\d+) of (\d+)", out.stdout)}
        assert "ratio:" in out.stdout and len(got) == 5, out.stdout
        ent = [int(x) for x in re.findall(r"entries_after_\w+ (\d+)", out.stdout)]
        return got, ent

    n = gold["objects"]
    res = {"ours": [run(r["seed"]) for r in gold["runs"]],
           "ref": [({k: h / t for k, (h, t) in r["phases"].items()}, r["entries"]) for r in gold["runs"]]}
    for who in res:
        for got, ent in res[who]:
            assert got["read1"] == 1.0 and got["read2"] == 1.0, (who, got)     # nothing is evicted below capacity
            assert ent[0] == n and n - 64 <= ent[1] <= n + 4096, (who, ent)
    report = {}
    for phase in ("reput_new", "reput_old", "read4"):
        a = float(np.mean([g[phase] for g, _ in res["ours"]]))
        b = float(np.mean([g[phase] for g, _ in res["ref"]]))
        report[phase] = (round(100 * a, 2), round(100 * b, 2))
    print("exerciser hit ratios % (ours, reference):", report)
    for phase, (a, b) in report.items():
        assert abs(a - b) <= 2.0, report


@pytest.mark.gpu
def test_cache_directory_interchange_with_the_reference(E, gpu, oracle, tmp_path):
    """SURVEY.md §8 f3: a cache directory written by one implementation is readable by the other,
    through tools/snap2lmdb (test infrastructure that links the compiled reference; LMDB stays out of
    the product).  (1) pages put through the GPU path -> snapshot -> LMDB files -> the reference's
    cachemap_get returns them; (2) pages put through the reference -> LMDB files -> snapshot -> this
    library restores them on first use and cachemap_get returns them."""
    import ctypes as C
    import subprocess
    import sys
    R = oracle.ref()
    if R is None:
        pytest.skip("oracle/_ref was not built")
    sys.path.insert(0, os.path.dirname(__file__))
    from test_oracle_pin import _build_snap2lmdb
    exe = _build_snap2lmdb(tmp_path)
    n = 48
    pages = np.stack([datagen.make_page("RTZMPAX"[i % 7], 65536, 300 + i) for i in range(n)])
    off = np.arange(n, dtype=np.uint64) << np.uint64(16)
    nh = np.full(n, 4242, dtype=np.uint64)
    gen = np.full(n, 5, dtype=np.uint32)
    # (1) GPU -> reference
    d_gpu, d_lmdb = tmp_path / "gpu", tmp_path / "lmdb"
    d_gpu.mkdir(); d_lmdb.mkdir()
    cm = E.Cachemap(str(d_gpu), 2048, 12, 16)
    cm.put_batch(off, nh, gen, pages)
    assert cm.checkpoint() == 0
    cm.free()
    snap = str(d_gpu / "cachemap_b200.snap")
    out = subprocess.run([exe, "to-lmdb", snap, str(d_lmdb), "2048", "16"], capture_output=True, text=True)
    assert out.returncode == 0 and f"{n} of {n}" in out.stdout, out.stdout + out.stderr
    # The reference's library runs in child processes under a watchdog: its cachemap_create starts the
    # put threads before it initialises their mutex and condition variable (cachemap.c:123-138) and a
    # process that loses that race never gets going; such a child is killed and started again.
    np.save(tmp_path / "pages.npy", pages)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def reference_child(body: str):
        code = ("import sys, ctypes as C, numpy as np\n"
                f"sys.path.insert(0, {root!r})\n"
                "from oracle import ef_oracle as O\n"
                "R = O.ref()\n"
                f"pages = np.load({str(tmp_path / 'pages.npy')!r}); n = len(pages)\n"
                "off = np.arange(n, dtype=np.uint64) << np.uint64(16)\n" + body + "\nprint('child ok', flush=True)\nimport os; os._exit(0)\n")
        for attempt in range(6):
            try:
                r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60)
            except subprocess.TimeoutExpired:
                continue
            assert r.returncode == 0 and "child ok" in r.stdout, r.stdout + r.stderr
            return
        raise AssertionError("the reference library hung at start-up in every attempt")

    reference_child(
        f"rcm = R.cachemap_create({str(d_lmdb)!r}.encode(), 2048, 12, 16)\n"
        "for i in range(n):\n"
        "    p = R.cachemap_get(rcm, int(off[i]), 4242, 5)\n"
        "    assert p and bytes((C.c_uint8 * 65536).from_address(p)) == pages[i].tobytes(), i\n")
    # (2) reference -> GPU
    d_ref, d_back = tmp_path / "ref", tmp_path / "back"
    d_back.mkdir()
    reference_child(
        "import shutil, os\n"
        f"shutil.rmtree({str(d_ref)!r}, ignore_errors=True); os.mkdir({str(d_ref)!r})\n"
        f"rcm2 = R.cachemap_create({str(d_ref)!r}.encode(), 2048, 12, 16)\n"
        "for i in range(n):\n"
        "    R.cachemap_put(rcm2, int(off[i]), 99, 7, pages[n - 1 - i].ctypes.data)\n")
    out = subprocess.run([exe, "from-lmdb", str(d_ref), str(d_back / "cachemap_b200.snap"), "16"], capture_output=True, text=True)
    assert out.returncode == 0 and f"{n} records" in out.stdout, out.stdout + out.stderr
    cm2 = E.Cachemap(str(d_back), 2048, 12, 16)
    got, hit = cm2.get_batch(off, np.full(n, 99, dtype=np.uint64), np.full(n, 7, dtype=np.uint32))
    assert hit.all() and (got == pages[::-1]).all()
    cm2.free()


@pytest.mark.gpu
def test_compaction_rebuilds_a_table_full_of_tombstones(E, gpu):
    """Linear probing never returns a slot: after many deletes the table is mostly tombstones.
    cmb200_compact then rebuilds it; every live key, its record, timestamp order and the counters
    survive, deleted keys stay deleted, and new keys can be put afterwards."""
    eng = E.Engine(pshift=12, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=512, flags=E.FINGERPRINT)
    assert eng.stats()["table_slots"] == 4096
    pages = np.stack([datagen.make_page("T", 4096, i) for i in range(512)])
    keep_u = np.full(300, 3, dtype=np.uint64); keep_l = np.arange(300, dtype=np.uint64)
    eng.put(keep_u, keep_l, pages[:300], ts=np.arange(300, dtype=np.uint64) + 1)
    for rnd in range(8):                                   # 8 x 400 keys put and deleted again
        u = np.full(400, 100 + rnd, dtype=np.uint64); l = np.arange(400, dtype=np.uint64)
        eng.put(u, l, pages[:400]); eng.unset(u, l)
    before = eng.stats()
    assert before["tombstones"] > 4096 // 8 and before["entries"] == 300
    fps0, ok0 = eng.read_fingerprints(keep_u, keep_l)
    eng.compact()
    after = eng.stats()
    assert after["tombstones"] == 0 and after["entries"] == 300 and after["arena_garbage"] == 0
    out, st = eng.get(keep_u, keep_l)
    assert (st == E.HIT).all() and (out == pages[:300]).all()
    out, st = eng.get_small(keep_u, keep_l)
    assert (st == E.HIT).all() and (out == pages[:300]).all()
    fps1, ok1 = eng.read_fingerprints(keep_u, keep_l)
    assert (ok0 == ok1).all() and (fps0 == fps1).all()
    _, st = eng.get(np.full(400, 103, dtype=np.uint64), np.arange(400, dtype=np.uint64))
    assert (st == E.MISS).all()
    u = np.full(200, 500, dtype=np.uint64); l = np.arange(200, dtype=np.uint64)
    eng.put(u, l, pages[200:400])
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and (out == pages[200:400]).all() and eng.stats()["entries"] == 500
    eng.close()


@pytest.mark.gpu
def test_small_get_walks_records_with_and_without_checkpoints(E, gpu, oracle, tmp_path, monkeypatch):
    """k_get_small parses a record in 16 sections when the encoder left checkpoints for it and with
    one warp otherwise (engine without the side table, records loaded from a snapshot, records moved
    by a compaction): the pages must be the same bytes either way, for every content class and for
    ragged compressibility (checkpoint sections that are empty, a page that is ONE sequence)."""
    bs = 65536
    kinds = "RTZMPAX"
    n = 84
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], bs, 900 + i) for i in range(n)])
    pages[3, :] = 0                                            # one match over the whole page
    pages[4, :40000] = 7                                       # long run, then noise
    u = np.full(n, 77, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)

    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.put(u, l, pages)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    # stored blocks are the reference's bytes, so the oracle decodes them to the same pages
    snap = str(tmp_path / "ck.snap")
    eng.save(snap)
    # compaction moves the records: their checkpoints no longer name them (one-warp walk), same pages
    eng.unset(u[:10], l[:10])
    eng.compact()
    out, st = eng.get_small(u, l)
    assert (st[:10] == E.MISS).all() and (st[10:] == E.HIT).all() and (out[10:] == pages[10:]).all()
    # rewriting a key renews its checkpoints
    eng.put(u[10:20], l[10:20], pages[30:40])
    out, st = eng.get_small(u[10:20], l[10:20])
    assert (st == E.HIT).all() and (out == pages[30:40]).all()
    eng.close()

    # records that arrive from a snapshot have no checkpoints
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.load(snap)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.close()

    # an engine without the side table
    monkeypatch.setenv("CMB200_CKPT", "0")
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.put(u, l, pages)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.close()


@pytest.mark.gpu
def test_small_get_in_two_halves(E, gpu):
    """cmb200_get_small_begin / _end: the statuses appear one by one in the ticket's page-locked
    words (PENDING until then), a page is complete once its status is, and end may run on another
    thread than begin."""
    import ctypes as C
    import threading
    bs = 65536
    kinds = "RTZM"
    n = 24
    pages = np.stack([datagen.make_page(kinds[i % 4], bs, 40 + i) for i in range(n)])
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    u = np.full(n, 5, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    eng.put(u, l, pages)
    L = E.lib()

    class Ticket(C.Structure):
        _fields_ = [("lane", C.c_int), ("n", C.c_uint32), ("status", C.POINTER(C.c_int32))]

    addr = np.stack([np.append(u, 6), np.append(l, 0)], axis=1).astype(np.uint64).copy()   # last one misses
    m = n + 1
    buf = L.cmb200_host_alloc(m * bs)
    for rounds in range(3):
        t = Ticket()
        assert L.cmb200_get_small_begin(eng.h, m, addr.ctypes.data, buf, C.byref(t)) == 0
        assert t.lane >= 0 and t.n == m
        got = np.zeros(m, dtype=bool)
        arr = np.ctypeslib.as_array((C.c_uint8 * (m * bs)).from_address(buf)).reshape(m, bs)
        while not got.all():
            for i in range(m):
                if not got[i] and t.status[i] != -1:
                    # the page is there as soon as its status is
                    if i < n:
                        assert t.status[i] == E.HIT and (arr[i] == pages[i]).all()
                    else:
                        assert t.status[i] == E.MISS
                    got[i] = True
        st = np.zeros(m, dtype=np.int32)
        rc = []
        th = threading.Thread(target=lambda: rc.append(L.cmb200_get_small_end(eng.h, C.byref(t), st.ctypes.data)))
        th.start()
        th.join()
        assert rc == [0] and t.lane == -1
        assert (st[:n] == E.HIT).all() and st[n] == E.MISS
    # more launches in flight than the engine has lanes: begin waits for a lane, nothing is lost
    tickets = []
    bufs = []

    def one(i):
        b = L.cmb200_host_alloc(bs)
        t = Ticket()
        a = addr[i:i + 1].copy()
        assert L.cmb200_get_small_begin(eng.h, 1, a.ctypes.data, b, C.byref(t)) == 0
        s1 = np.zeros(1, dtype=np.int32)
        assert L.cmb200_get_small_end(eng.h, C.byref(t), s1.ctypes.data) == 0
        page = np.ctypeslib.as_array((C.c_uint8 * bs).from_address(b)).copy()
        L.cmb200_host_free(b)
        tickets.append((i, int(s1[0]), page))

    ths = [threading.Thread(target=one, args=(i % n,)) for i in range(96)]
    [x.start() for x in ths]
    [x.join() for x in ths]
    assert len(tickets) == 96
    for i, s1, page in tickets:
        assert s1 == E.HIT and (page == pages[i]).all()
    L.cmb200_host_free(buf)
    eng.close()
