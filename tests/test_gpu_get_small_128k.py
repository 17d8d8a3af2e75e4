"""GPU tests of the fused single-page get at 128 KiB pages (pshift 17), where k_get_small_pair decodes
each request in a cluster of two CTAs (record in one, page in the other).  Every answer is checked
against cmb200_get_batch, which has its own decoder (k_decode), or against the pages that were put."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import datagen

pytestmark = pytest.mark.gpu
PSHIFT = 17
BS = 1 << PSHIFT


@pytest.fixture(autouse=True)
def small_engine(monkeypatch):
    monkeypatch.setenv("CMB200_ARENA_MB", "512")
    monkeypatch.setenv("CMB200_MAX_BATCH", "512")
    monkeypatch.setenv("CMB200_PERSIST", "0")


def _pages(n, seed):
    """Every content class, plus the pages whose lengths need the wide descriptor fields."""
    kinds = "RTZMPAX"
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], BS, seed + i) for i in range(n)])
    pages[0, :] = 0                                   # ONE match of ~131 KiB
    pages[1, :70000] = 9                              # a match longer than 65 535, then noise
    pages[2, :] = datagen.make_page("R", BS, seed + 7777)
    pages[2, 80 * 1024:] = 0                          # a literal run above 65 536, then one long match
    return pages


def _keys(n, u0):
    return np.full(n, u0, dtype=np.uint64), np.arange(n, dtype=np.uint64)


def test_same_answers_as_the_batch_get(E, gpu):
    n = 40
    pages = _pages(n, 100)
    for accel in (12, 0):                             # LZ4 records / raw pages
        eng = E.Engine(pshift=PSHIFT, accel=accel, capacity=4096, arena_bytes=128 << 20, max_batch=64)
        u, l = _keys(n, 31)
        eng.put(u, l, pages)
        qu = np.concatenate([u, np.full(5, 32, dtype=np.uint64)])
        ql = np.concatenate([l, np.arange(5, dtype=np.uint64)])   # 5 misses
        out_b, st_b = eng.get(qu, ql)
        out_s, st_s = eng.get_small(qu, ql)
        assert (st_s == st_b).all() and (st_s[:n] == E.HIT).all() and (st_s[n:] == E.MISS).all()
        assert (out_s[:n] == pages).all() and (out_b[:n] == pages).all()
        eng.put(u[:10], l[:10], pages[10:20])         # a rewrite is served from its new record
        eng.unset(u[20:25], l[20:25])                 # an unset key misses
        out_b, st_b = eng.get(u, l)
        out_s, st_s = eng.get_small(u, l)
        assert (st_s == st_b).all() and (st_s[20:25] == E.MISS).all()
        want = pages.copy()
        want[:10] = pages[10:20]
        hit = st_s == E.HIT
        assert hit.sum() == n - 5 and (out_s[hit] == want[hit]).all()
        eng.close()


def test_with_and_without_checkpoints(E, gpu, tmp_path, monkeypatch):
    """Sections from the encoder's checkpoints (fresh puts) and the one-warp walk (records moved by
    compaction, loaded from a snapshot, an engine without the side table) give the same pages."""
    n = 42
    pages = _pages(n, 900)
    u, l = _keys(n, 77)
    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64)
    eng.put(u, l, pages)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    snap = str(tmp_path / "ck.snap")
    eng.save(snap)
    eng.unset(u[:10], l[:10])
    eng.compact()
    out, st = eng.get_small(u, l)
    assert (st[:10] == E.MISS).all() and (st[10:] == E.HIT).all() and (out[10:] == pages[10:]).all()
    eng.put(u[10:20], l[10:20], pages[30:40])         # rewrites get checkpoints again
    out, st = eng.get_small(u[10:20], l[10:20])
    assert (st == E.HIT).all() and (out == pages[30:40]).all()
    eng.close()

    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64)
    eng.load(snap)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.close()

    monkeypatch.setenv("CMB200_CKPT", "0")
    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64)
    eng.put(u, l, pages)
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.close()


def _first_offset_at(block: bytes) -> int:
    """Block offset of the first sequence's match offset."""
    tok = block[0]
    ip, lit = 1, tok >> 4
    if lit == 15:
        while True:
            b = block[ip]
            ip += 1
            lit += b
            if b != 255:
                break
    return ip + lit


def test_malformed_stored_blocks(E, gpu, oracle, tmp_path):
    """Blocks altered with valid lengths, loaded from a snapshot written by oracle/snapshot.py: the
    fused get answers like the batch get (BAD_DECODE or HIT), with the same page where it is a HIT."""
    from oracle import snapshot
    n = 28
    pages = _pages(n, 4242)
    u, l = _keys(n, 55)
    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64)
    eng.put(u, l, pages)
    recs = eng.read_records(u, l)
    eng.close()
    rng = np.random.default_rng(17)
    out_recs = []
    for i, rec in enumerate(recs):
        prefix, blk = bytearray(rec[:24]), bytearray(rec[24:])
        clen = int.from_bytes(prefix[16:20], "little")
        assert clen == len(blk) and clen > 0
        kind = i % 4
        if kind == 0:                                 # an offset that points before the page
            at = _first_offset_at(bytes(blk))
            if at + 2 <= len(blk):
                blk[at:at + 2] = (0xffff).to_bytes(2, "little")
        elif kind == 1:                               # length bytes: token nibbles and extension bytes
            blk[0] = 0xff
            if len(blk) > 1:
                blk[1] = int(rng.integers(0, 256))
        elif kind == 2:                               # truncated last literals
            blk = blk[:-3]
        else:                                         # a few random bytes
            for p in rng.integers(0, len(blk), 4):
                blk[int(p)] = int(rng.integers(0, 256))
        prefix[16:20] = len(blk).to_bytes(4, "little")
        out_recs.append((i + 1, 0, 0, bytes(prefix + blk)))
    path = str(tmp_path / "bad.snap")
    snapshot.write_snapshot(path, PSHIFT, out_recs)
    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64)
    assert eng.load(path) == n
    out_b, st_b = eng.get(u, l)
    out_s, st_s = eng.get_small(u, l)
    assert (st_s == st_b).all(), (st_s, st_b)
    assert set(st_s.tolist()) <= {E.HIT, E.BAD_DECODE} and (st_s == E.BAD_DECODE).any()
    hit = st_s == E.HIT
    assert (out_s[hit] == out_b[hit]).all()
    eng.close()


def test_host_tier(E, gpu):
    n = 40
    pages = _pages(n, 300)
    u, l = _keys(n, 41)
    eng = E.Engine(pshift=PSHIFT, accel=12, capacity=4096, arena_bytes=128 << 20, max_batch=64,
                   host_tier_bytes=64 << 20)
    eng.put(u, l, pages)
    assert eng.demote(u[::2], l[::2]) == n // 2
    h0 = eng.host_tier_stats()["hits"]
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    assert eng.host_tier_stats()["hits"] - h0 == n // 2
    out, st = eng.get_small(u[:7], l[:7])             # 4 of them in the tier
    assert (st == E.HIT).all() and (out == pages[:7]).all()
    assert eng.host_tier_stats()["hits"] - h0 == n // 2 + 4
    eng.close()


def test_small_gets_overlap_puts_without_torn_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 128, 131072
eng = E.Engine(pshift=17, accel=12, capacity=8192, arena_bytes=3 << 30, max_batch=256)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 77, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
la = eng.put(u, l, A)
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
    lb = eng.put(u, l, B if rnd % 2 == 0 else A)
stop.set(); [t.join() for t in th]
assert not bad, bad
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
assert (la != eng.put(u, l, B)).any()          # the two contents have records of different sizes
print("no torn pages", gets[0])
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def test_drop_in_gets_take_the_fused_path(E, gpu, oracle, tmp_path):
    """cachemap_get / cachemap_read_range at pshift 17 from several threads: right pages, counters as
    the reference counts them, and no k_decode launch (the fallback through cmb200_get_batch)."""
    n = 96
    pages = _pages(n, 5150)
    cm = E.Cachemap(str(tmp_path), 4096, 12, PSHIFT)
    assert cm.ok
    nh = np.full(n, 6, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    off = np.arange(n, dtype=np.uint64) << np.uint64(PSHIFT)
    cm.put_batch(off, nh, gen, pages)
    h = cm.engine_handle()
    rq0, ht0 = cm.counters()
    launches0 = E.engine_stats(h)["decode_kernel_launches"]
    errors = []

    def worker(t):
        try:
            for i in range(t, n, 8):
                got = cm.get(int(off[i]), 6, 0)
                if got != pages[i].tobytes():
                    errors.append(("get", i))
                if cm.get(int(off[i]), 7, 0) is not None:          # another file: a miss
                    errors.append(("miss", i))
            base = 12 * t
            got = cm.read_range(6, 0, base * BS, 4 * BS)
            if got != pages[base:base + 4].tobytes():
                errors.append(("range", base))
        except Exception as e:                                      # pragma: no cover
            errors.append(repr(e))

    th = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errors, errors[:8]
    rq, ht = cm.counters()
    assert rq - rq0 == 2 * n + 8 * 4 and ht - ht0 == n + 8 * 4, (rq - rq0, ht - ht0)
    assert E.engine_stats(h)["decode_kernel_launches"] == launches0
    cm.free()
