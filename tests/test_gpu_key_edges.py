"""The CUDA store on addresses that share a store key and on addresses whose key is the table's empty (0)
or tombstone (~0) marker (tests/golden/key_edges.json).

The store keeps one record per FNV-1a-64 key of the 16-byte address.  Two addresses with one key reach
the address compares of every lookup (k_lookup, the fused get's record-prefix check, k_unset, the
last-writer-wins of a put batch, k_import_records).  Keys 0 and ~0 are the table's own empty and
tombstone markers: their records live in side slots after the table, which every table walk (sampling,
export for snapshots and compaction, the rebuild, the fingerprint and checkpoint side tables, the host
tier) must treat as live records."""
import ctypes

import numpy as np
import pytest

import key_edges as K
from ckpt_def import ckpt_words

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return K.load()


def _ua(addrs):
    return (np.array([a[0] for a in addrs], dtype=np.uint64), np.array([a[1] for a in addrs], dtype=np.uint64))


# ---- the drop-in against the reference's answers ----------------------------------------------------

def _pages_ptr(cm):
    return ctypes.cast(cm.h, ctypes.POINTER(ctypes.c_void_p))[0]        # struct cachemap { pages, ...


def _bad_entries(capfd):
    """`bad entry` lines the drop-in printed since the last call (C stdio is flushed first)."""
    ctypes.CDLL(None).fflush(None)
    return capfd.readouterr().out.count("bad entry")


@pytest.mark.parametrize("slots", [None, "0"])
@pytest.mark.parametrize("pshift", (12, 16, 17))
def test_drop_in_replays_the_reference(E, gpu, fx, tmp_path, monkeypatch, capfd, pshift, slots):
    """cachemap_put / cachemap_get / filemap_unset over colliding and sentinel-key addresses answer as
    the reference did, page, miss or bad entry per get, with the write-behind ring and without; then
    put A / put B / get A, back to back, misses with a bad entry every round, whatever the flusher has
    landed by then."""
    monkeypatch.setenv("CMB200_ARENA_MB", "512")
    monkeypatch.setenv("CMB200_PERSIST", "0")
    if slots is None:
        monkeypatch.delenv("CMB200_WB_SLOTS", raising=False)
    else:
        monkeypatch.setenv("CMB200_WB_SLOTS", slots)
    run = fx["runs"][str(pshift)]
    cm = E.Cachemap(str(tmp_path), fx["capacity"], fx["accel"], pshift)
    assert cm.ok
    unset = E.lib().filemap_unset
    _bad_entries(capfd)
    gets = []
    for kind, u, l, content in fx["ops"]:
        off, nh, gen = K.cachemap_args(u, l, pshift)
        if kind == "put":
            cm.put(off, nh, gen, K.page(content, pshift))
        elif kind == "unset":
            unset(_pages_ptr(cm), (ctypes.c_uint64 * 2)(u, l))
        else:
            p = cm.get(off, nh, gen)
            bad = _bad_entries(capfd)
            assert bad <= (p is None), (u, l)
            gets.append(K.sha(p) if p is not None else "bad entry" if bad else "miss")
    for i, (g, w) in enumerate(zip(gets, run["gets"])):
        assert g == w, f"get #{i}: {g}, the reference {w}"
    assert len(gets) == len(run["gets"])
    assert cm.counters() == (run["requests"], run["hits"])
    assert E.lib().filemap_entries(_pages_ptr(cm)) == run["entries"]

    a, b = fx["groups"]["quad"][:2]
    pa, pb = K.page(["T", 1], pshift), K.page(["M", 2], pshift)
    rounds = 200
    rq0, ht0 = cm.counters()
    _bad_entries(capfd)
    for _ in range(rounds):
        cm.put(*K.cachemap_args(*a, pshift), pa)
        cm.put(*K.cachemap_args(*b, pshift), pb)
        assert cm.get(*K.cachemap_args(*a, pshift)) is None
    assert _bad_entries(capfd) == rounds
    assert cm.counters() == (rq0 + rounds, ht0)
    assert cm.get(*K.cachemap_args(*b, pshift)) == pb.tobytes()
    cm.free()


# ---- the engine against the store model -------------------------------------------------------------

_STATUS = {"hit": "HIT", "miss": "MISS", "bad entry": "BAD_ENTRY"}


def _check_against_model(E, O, eng, model, universe, pshift):
    u, l = _ua(universe)
    recs = eng.read_records(u, l)
    for i, a in enumerate(universe):
        r = model.rec.get(O.addr_key(*a))
        want = model.record_bytes(*a) if r is not None and r[0] == a else None
        assert recs[i] == want, (i, a)
    want = [model.get_status(*K.cachemap_args(*a, pshift)) for a in universe]
    for name, (out, st) in (("get", eng.get(u, l)), ("get_small", eng.get_small(u, l))):
        for i, (ws, wp) in enumerate(want):
            assert st[i] == getattr(E, _STATUS[ws]), (name, i, universe[i], int(st[i]), ws)
            if wp is not None:
                assert out[i].tobytes() == bytes(wp), (name, i)
    assert eng.entries() == model.entries()


@pytest.mark.parametrize("pshift", (12, 16, 17))
def test_engine_resolves_colliding_keys_like_the_model(E, gpu, oracle, fx, pshift):
    """Put batches with members of one key in one batch (both orders), across a max_batch boundary and
    next to sentinel-key addresses: the stored records, the -1 lens of superseded chunks, HIT /
    BAD_ENTRY / MISS of both gets (k_get_small at 4 and 64 KiB, k_get_small_pair at 128 KiB), unset
    through another member and the put after it, as the store model has them."""
    g, o = fx["groups"], fx["ordinary"]
    q, k0, k1, p0, p1 = g["quad"], g["key0"], g["key_ones"], g["pair0"], g["pair1"]
    universe = [a for grp in g.values() for a in grp] + o
    mb = 8
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=256 << 20, max_batch=mb)
    model = oracle.StoreModel(pshift, 12)
    seed = [0]

    def put(rows):
        pages = np.stack([K.page(["TMRXZ"[i % 5], 300 + i], pshift) for i in range(seed[0], seed[0] + len(rows))])
        seed[0] += len(rows)
        lens = eng.put(*_ua(rows), pages)
        keys = [oracle.addr_key(*a) for a in rows]
        for i, a in enumerate(rows):
            model.put(*K.cachemap_args(*a, pshift), pages[i])
            superseded = any(keys[j] == keys[i] for j in range(i + 1, min(len(rows), (i // mb + 1) * mb)))
            assert lens[i] == (-1 if superseded else len(oracle.lz4_encode(pages[i], 12))), (i, a)
        _check_against_model(E, oracle, eng, model, universe, pshift)

    put([q[0], q[1], o[0], k0[0], k1[0], p0[0]])                    # A then B in one batch
    put([q[1], q[0], k0[1], k0[0], p0[1], o[1], k1[1]])             # B then A, sentinels both orders
    put([o[2], o[3], o[4], o[5], k1[2], o[1], k0[2], q[2],          # q[2] | q[3] across the boundary
         q[3], k0[1], k1[0], p1[0], p1[1]])
    for via in (q[0], k0[0], k1[1], p1[0]):                          # unset through another member
        eng.unset(*_ua([via]))
        model.unset(*via)
        _check_against_model(E, oracle, eng, model, universe, pshift)
    put([q[1], k0[2], k1[2], p1[1]])                                 # stored again after the unset
    assert eng.stats()["dropped_puts"] == 0
    eng.close()


# ---- the side slots of keys 0 and ~0 through every table walk ----------------------------------------

def _side(fx):
    return [fx["groups"]["key0"][0], fx["groups"]["key_ones"][0]]


def _expect_side(E, eng, side, pages, fps=None):
    u, l = _ua(side)
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and (out == pages).all(), st
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all(), st
    if fps is not None:
        f, ok = eng.read_fingerprints(u, l)
        assert (ok == 1).all() and (f == fps).all()


def test_sentinel_keys_survive_compaction_snapshots_and_the_table_rebuild(E, gpu, oracle, fx, tmp_path):
    """Records under key 0 and key ~0 stay readable and unchanged through compact(), save and load into
    an engine of another geometry, and the tombstone-driven table rebuild, with their fingerprints and
    parse checkpoints."""
    side = _side(fx)
    su, sl = _ua(side)
    pages = np.stack([K.page(["T", 11], 12), K.page(["X", 12], 12)])
    eng = E.Engine(pshift=12, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=512,
                   flags=E.FINGERPRINT)
    eng.put(su, sl, pages, ts=np.array([5, 6], dtype=np.uint64))
    recs0 = eng.read_records(su, sl)
    for i, a in enumerate(side):
        blk = oracle.lz4_encode(pages[i], 12)
        assert recs0[i] == oracle.record_prefix(a[0], a[1], len(blk)) + blk
    fps = np.array([oracle.fingerprint128(p) for p in pages], dtype=np.uint64)
    _expect_side(E, eng, side, pages, fps)

    filler = K.page(["M", 13], 12)
    fu, fl = np.full(64, 77, dtype=np.uint64), np.arange(64, dtype=np.uint64)
    eng.put(fu, fl, np.stack([filler] * 64))
    eng.unset(fu[::2], fl[::2])
    assert eng.compact() > 0                                         # records moved past the garbage
    assert eng.read_records(su, sl) == recs0
    _expect_side(E, eng, side, pages, fps)

    path = str(tmp_path / "side.snap")
    assert eng.save(path) == 2 + 32
    other = E.Engine(pshift=12, accel=12, capacity=65536, arena_bytes=128 << 20, max_batch=64, flags=E.FINGERPRINT)
    assert other.load(path) == 2 + 32 and other.entries() == 2 + 32
    assert other.read_records(su, sl) == recs0
    _expect_side(E, other, side, pages, fps)
    other.close()

    for rnd in range(8):                                             # 8 x 400 keys put and deleted again
        u, l = np.full(400, 100 + rnd, dtype=np.uint64), np.arange(400, dtype=np.uint64)
        eng.put(u, l, np.stack([filler] * 400))
        eng.unset(u, l)
    assert eng.stats()["tombstones"] > 4096 // 8
    eng.compact()
    assert eng.stats()["tombstones"] == 0 and eng.entries() == 2 + 32  # the table was rebuilt
    assert eng.read_records(su, sl) == recs0
    _expect_side(E, eng, side, pages, fps)
    words, ok = eng.read_checkpoints(su, sl)
    assert (ok == 1).all(), ok
    for i, r in enumerate(recs0):
        assert words[i, 1:].tolist() == ckpt_words(r[24:], 4096)[1:]
    eng.unset(su, sl)
    _, st = eng.get(su, sl)
    assert (st == E.MISS).all() and eng.entries() == 32
    eng.close()


def test_sentinel_keys_through_the_host_tier_verify_and_sampling(E, gpu, oracle, fx):
    """Key 0 and key ~0 records go to the host tier and back, are counted as verified by
    verify_store, and are what sample() returns on a table that holds nothing else (the bounded walk
    fails and k_sample_scan finds them); once unset, sample() finds nothing."""
    side = _side(fx)
    su, sl = _ua(side)
    pages = np.stack([K.page(["R", 21], 16), K.page(["T", 22], 16)])
    eng = E.Engine(pshift=16, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, host_tier_bytes=16 << 20,
                   flags=E.VERIFY)
    eng.put(su, sl, pages, ts=np.array([40, 41], dtype=np.uint64))
    recs0 = eng.read_records(su, sl)
    assert eng.demote(su, sl) == 2
    assert eng.host_tier_stats()["records"] == 2
    assert eng.read_records(su, sl) == recs0
    _expect_side(E, eng, side, pages)
    assert eng.promote(su, sl) == 2
    assert eng.host_tier_stats()["records"] == 0 and eng.read_records(su, sl) == recs0
    _expect_side(E, eng, side, pages)
    _, _, n_bad, checked = eng.verify_store()
    assert n_bad == 0 and checked == 2

    r = np.arange(256, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    addr, ts, ok = eng.sample(r)
    assert (ok == 1).all(), ok
    got = {(int(a[0]), int(a[1]), int(t)) for a, t in zip(addr, ts)}
    assert got <= {(side[0][0], side[0][1], 40), (side[1][0], side[1][1], 41)}
    eng.unset(su, sl)
    _, _, ok = eng.sample(r)
    assert (ok == 0).all() and eng.entries() == 0
    eng.close()


# ---- a record imported from another rank against a local one of the same key ------------------------

@pytest.mark.parametrize("remote_newer", [True, False])
def test_import_of_a_colliding_record_keeps_the_newer(E, gpu, fx, remote_newer):
    """A put locally through put_step, B (same key) imported from another rank through
    import_records_dev: the newer stream position wins, and the loser's address misses."""
    from edge_fuse_b200 import sharding
    a, b = fx["groups"]["quad"][:2]
    world, rank, base = 4, 1, 1000
    eng = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64, flags=E.FINGERPRINT)
    page = K.page(["T", 31], 12)
    d_rec = eng.dev_alloc(32)
    eng.set_stream_order(base + rank, world)
    eng.wait(eng.put_step(*_ua([a]), page[None], rank=rank, records_dev=d_rec))
    eng.sync()
    pos_b = base + 10 if remote_newer else 3
    rows = sharding.pack_records([b[0]], [b[1]], [pos_b], 2, [200], rec_off=[4096])
    d_rows = eng.dev_alloc(rows.nbytes)
    eng.h2d(d_rows, rows)
    eng.import_records_dev(len(rows), d_rows, rank)
    eng.sync()
    status, owner = eng.locate(*_ua([a, b]))
    winner, loser = (b, a) if remote_newer else (a, b)
    out, st = eng.get(*_ua([loser]))
    _, st_small = eng.get_small(*_ua([loser]))
    assert st[0] in (E.MISS, E.BAD_ENTRY) and st_small[0] in (E.MISS, E.BAD_ENTRY), (st, st_small)
    if remote_newer:
        assert status[1] == E.REMOTE and owner[1] == 2 and status[0] in (E.MISS, E.BAD_ENTRY), status
        assert eng.stats()["remote_entries"] == 1 and eng.entries() == 0
    else:
        assert status[0] == E.HIT and status[1] in (E.MISS, E.BAD_ENTRY), status
        out, st = eng.get(*_ua([winner]))
        _, st_small = eng.get_small(*_ua([winner]))
        assert st[0] == E.HIT and st_small[0] == E.HIT and (out[0] == page).all()
        assert eng.stats()["remote_entries"] == 0 and eng.entries() == 1
    for p in (d_rec, d_rows):
        eng.dev_free(p)
    eng.close()
