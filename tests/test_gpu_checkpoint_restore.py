"""GPU tests of the parse checkpoints that k_get_small splits a record's token chain with: the encoder's
words equal ckpt_def.ckpt_words of the stored block, and records keep bit-equal words when they are
loaded from a snapshot (rebuilt from the block by k_restore), moved by a compaction, carried through a
table rebuild or demoted to the host tier.  Blocks whose chain does not fit get none; every answer of
the fused get stays the batch get's."""
import os
import subprocess
import sys

import numpy as np
import pytest

import datagen
from ckpt_def import ckpt_words

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pages(n, bs, seed):
    """Every content class, plus a zero page (one match) and a long run followed by noise."""
    kinds = "RTZMPAX"
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], bs, seed + i) for i in range(n)])
    pages[3, :] = 0
    pages[4, :bs * 5 // 8] = 7
    return pages


def _keys(n, u0):
    return np.full(n, u0, dtype=np.uint64), np.arange(n, dtype=np.uint64)


def _block_words(eng, u, l, bs):
    """ckpt_words of each stored block (None for a raw page or a chain that does not fit)."""
    out = []
    for r in eng.read_records(u, l):
        clen = int.from_bytes(r[16:20], "little")
        out.append(ckpt_words(r[24:], bs) if clen else None)
    return out


@pytest.mark.parametrize("accel", [12, 20])
@pytest.mark.parametrize("pshift", [6, 10, 12, 14, 16, 17])
def test_encoder_words_equal_the_definition(E, gpu, pshift, accel):
    bs, n = 1 << pshift, 16
    pages = _pages(n, bs, 100 * pshift + accel)
    u, l = _keys(n, 5)
    eng = E.Engine(pshift=pshift, accel=accel, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.put(u, l, pages)
    words, ok = eng.read_checkpoints(u, l)
    assert (ok == 1).all(), ok
    for i, w in enumerate(_block_words(eng, u, l, bs)):
        assert w is not None and words[i, 1:].tolist() == w[1:], (i, words[i].tolist(), w)
    _, ok = eng.read_checkpoints(u, l + np.uint64(1000))
    assert (ok == -1).all()                                    # absent keys
    eng.close()


@pytest.mark.parametrize("pshift", [12, 16, 17])
def test_load_rebuilds_the_encoders_words(E, gpu, tmp_path, pshift):
    bs, n = 1 << pshift, 28
    pages = _pages(n, bs, 700 + pshift)
    u, l = _keys(n, 9)
    geo = dict(pshift=pshift, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    for accel in (12, 0):
        eng = E.Engine(accel=accel, **geo)
        eng.put(u, l, pages)
        w0, ok0 = eng.read_checkpoints(u, l)
        path = str(tmp_path / f"a{accel}.snap")
        assert eng.save(path) == n
        eng.close()
        eng = E.Engine(accel=accel, **geo)
        assert eng.load(path) == n
        w1, ok1 = eng.read_checkpoints(u, l)
        if accel:
            assert (ok0 == 1).all() and (ok1 == 1).all(), ok1
            assert (w1[:, 1:] == w0[:, 1:]).all()
        else:
            assert (ok0 == 0).all() and (ok1 == 0).all()       # raw pages have no checkpoints
        out, st = eng.get_small(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
        eng.close()


def test_compaction_moves_the_tag(E, gpu):
    bs, n = 65536, 84
    pages = _pages(n, bs, 4100)
    u, l = _keys(n, 13)
    eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.put(u, l, pages)
    w0, ok0 = eng.read_checkpoints(u, l)
    gone = np.arange(n) % 3 == 0
    eng.unset(u[gone], l[gone])
    assert eng.compact() > 0
    assert eng.stats()["tombstones"] > 0                       # no table rebuild in this one
    keep = ~gone
    w1, ok1 = eng.read_checkpoints(u[keep], l[keep])
    assert (ok1 == 1).all(), ok1
    assert (w1[:, 1:] == w0[keep, 1:]).all()
    assert (w1[:, 0] != w0[keep, 0]).any()                     # records did move
    out, st = eng.get_small(u, l)
    assert (st[gone] == E.MISS).all() and (st[keep] == E.HIT).all() and (out[keep] == pages[keep]).all()
    eng.close()


def test_table_rebuild_carries_the_side_table(E, gpu):
    eng = E.Engine(pshift=12, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=512)
    pages = _pages(512, 4096, 77)
    ku, kl = _keys(300, 3)
    eng.put(ku, kl, pages[:300])
    w0, ok0 = eng.read_checkpoints(ku, kl)
    for rnd in range(3):                                       # 3 x 400 keys put and deleted: > cap/8 tombstones
        u, l = _keys(400, 100 + rnd)
        eng.put(u, l, pages[:400])
        eng.unset(u, l)
    assert eng.stats()["tombstones"] > 4096 // 8
    eng.compact()
    assert eng.stats()["tombstones"] == 0                      # the table was rebuilt
    w1, ok1 = eng.read_checkpoints(ku, kl)
    assert (ok0 == 1).all() and (ok1 == 1).all(), ok1
    assert (w1[:, 1:] == w0[:, 1:]).all()
    out, st = eng.get_small(ku, kl)
    assert (st == E.HIT).all() and (out == pages[:300]).all()
    eng.close()


def test_load_into_an_engine_with_a_host_tier(E, gpu, tmp_path):
    n, bs = 600, 65536
    pages = _pages(n, bs, 1100)
    u, l = _keys(n, 8)
    geo = dict(pshift=16, accel=12, capacity=4096, max_batch=128)
    eng = E.Engine(arena_bytes=512 << 20, **geo)
    eng.put(u, l, pages)
    w0, _ = eng.read_checkpoints(u, l)
    path = str(tmp_path / "tier.snap")
    assert eng.save(path) == n
    eng.close()
    eng = E.Engine(arena_bytes=16 << 20, host_tier_bytes=256 << 20, **geo)   # the arena holds ~ 300 of them
    assert eng.load(path) == n and eng.stats()["dropped_puts"] == 0
    in_tier = eng.host_tier_stats()["records"]
    assert in_tier > 0
    w1, ok1 = eng.read_checkpoints(u, l)
    assert (ok1 == 1).all(), ok1
    assert (w1[:, 1:] == w0[:, 1:]).all()
    h0 = eng.host_tier_stats()["hits"]
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    assert eng.host_tier_stats()["hits"] - h0 == in_tier
    eng.close()


def _first_offset_at(block: bytes) -> int:
    """Block offset of the first sequence's match offset."""
    ip, lit = 1, block[0] >> 4
    if lit == 15:
        while True:
            b = block[ip]
            ip += 1
            lit += b
            if b != 255:
                break
    return ip + lit


@pytest.mark.parametrize("pshift", [12, 16])
def test_malformed_blocks(E, gpu, tmp_path, pshift):
    """Blocks altered with valid lengths (oracle/snapshot.py): a chain that does not fit gets no
    checkpoints, one that fits may get them; the fused get answers as the batch get either way."""
    from oracle import snapshot
    bs, n = 1 << pshift, 28
    pages = _pages(n, bs, 4242 + pshift)
    u, l = _keys(n, 55)
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    eng.put(u, l, pages)
    recs = eng.read_records(u, l)
    eng.close()
    rng = np.random.default_rng(pshift)
    out_recs, blocks = [], []
    for i, rec in enumerate(recs):
        prefix, blk = bytearray(rec[:24]), bytearray(rec[24:])
        kind = i % 4
        if kind == 0:                                 # an offset that points before the page: the chain fits
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
        blocks.append(bytes(blk))
    path = str(tmp_path / "bad.snap")
    snapshot.write_snapshot(path, pshift, out_recs)
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64)
    assert eng.load(path) == n
    words, ok = eng.read_checkpoints(u, l)
    fits = [ckpt_words(b, bs) for b in blocks]
    assert any(f is None for f in fits) and any(f is not None for f in fits)
    for i, f in enumerate(fits):
        if f is None:
            assert ok[i] == 0, i
        else:
            assert ok[i] == 1 and words[i, 1:].tolist() == f[1:], i
    out_b, st_b = eng.get(u, l)
    out_s, st_s = eng.get_small(u, l)
    assert (st_s == st_b).all(), (st_s, st_b)
    assert set(st_s.tolist()) <= {E.HIT, E.BAD_DECODE} and (st_s == E.BAD_DECODE).any()
    hit = st_s == E.HIT
    assert (out_s[hit] == out_b[hit]).all()
    eng.close()


def test_small_gets_overlap_loads_without_torn_pages(E, gpu, tmp_path):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs, d = 128, 65536, sys.argv[1]
geo = dict(pshift=16, accel=12, capacity=8192, arena_bytes=1 << 30, max_batch=256)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 77, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
snaps = []
for name, P in (("a", A), ("b", B)):
    e = E.Engine(**geo); e.put(u, l, P); snaps.append(os.path.join(d, name + ".snap")); e.save(snaps[-1]); e.close()
eng = E.Engine(**geo)
eng.load(snaps[0])
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
for rnd in range(24):
    eng.load(snaps[1 - rnd % 2])
stop.set(); [t.join() for t in th]
assert not bad, bad
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
_, ok = eng.read_checkpoints(u, l)
assert (ok == 1).all()
print("no torn pages", gets[0])
'''
    out = subprocess.run([sys.executable, "-c", code, str(tmp_path)], cwd=ROOT, capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def test_drop_in_restart_serves_loaded_records_with_checkpoints(E, gpu, tmp_path, monkeypatch):
    monkeypatch.setenv("CMB200_ARENA_MB", "256")
    monkeypatch.setenv("CMB200_MAX_BATCH", "512")
    monkeypatch.setenv("CMB200_PERSIST", "1")
    n, ps = 64, 16
    pages = _pages(n, 1 << ps, 6060)
    nh = np.full(n, 6, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    off = np.arange(n, dtype=np.uint64) << np.uint64(ps)
    cm = E.Cachemap(str(tmp_path), 4096, 12, ps)
    assert cm.ok
    cm.put_batch(off, nh, gen, pages)
    assert cm.checkpoint() == 0
    cm.free()
    cm = E.Cachemap(str(tmp_path), 4096, 12, ps)
    assert cm.get(int(off[0]), 6, 0) == pages[0].tobytes()    # the first get loads the directory's snapshot
    u, l = nh, off >> np.uint64(ps)
    _, ok = E.read_checkpoints(cm.engine_handle(), u, l)
    assert (ok == 1).all(), ok
    for i in range(1, n):
        assert cm.get(int(off[i]), 6, 0) == pages[i].tobytes()
    cm.free()
