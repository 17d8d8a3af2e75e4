"""GPU tests of the engine's lifetime: engines made, used through every optional resource and every
grown scratch buffer, and closed, again and again in one process.  Each cycle checks its results,
so a buffer freed too early, freed twice or left to the next engine shows as a wrong page or status."""
import numpy as np
import pytest

import datagen

pytestmark = pytest.mark.gpu
CYCLES = 3


def _pages(bs, n, seed):
    return np.stack([datagen.make_page("TRZMPA"[i % 6], bs, seed + i) for i in range(n)])


# (pshift, flags, parse checkpoints); 18 has no fused single-page get and no checkpoint table
CONFIGS = [(p, f, True) for p in (12, 16, 17, 18) for f in ("", "FINGERPRINT", "VERIFY")]
CONFIGS += [(16, "", False), (12, "VERIFY", False)]


@pytest.mark.parametrize("pshift,flags,ckpt", CONFIGS)
def test_engines_are_made_used_and_closed_again(E, gpu, monkeypatch, pshift, flags, ckpt):
    if not ckpt:
        monkeypatch.setenv("CMB200_CKPT", "0")
    bs, n, gone = 1 << pshift, 160, 140                  # 140 tombstones > 1024 slots / 8: the table is rebuilt
    fl = getattr(E, flags) if flags else 0
    pages = _pages(bs, n, 40 + pshift)
    for cycle in range(CYCLES):
        eng = E.Engine(pshift=pshift, accel=12, capacity=256, table_slots=1024, arena_bytes=64 << 20,
                       max_batch=64, flags=fl)
        u = np.full(n, 11 + cycle, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        out, st = eng.get(u, l)
        assert (st == E.HIT).all() and (out == pages).all(), cycle
        if pshift <= 17:
            out, st = eng.get_small(u, l)
            assert (st == E.HIT).all() and (out == pages).all(), cycle
        if fl:
            fps0, ok0 = eng.read_fingerprints(u[gone:], l[gone:])
        eng.read_checkpoints(u, l)
        eng.unset(u[:gone], l[:gone])
        assert eng.stats()["tombstones"] > 1024 // 8
        eng.compact()
        s = eng.stats()
        assert s["tombstones"] == 0 and s["entries"] == n - gone and s["arena_garbage"] == 0, (cycle, s)
        out, st = eng.get(u, l)
        assert (st[:gone] == E.MISS).all() and (st[gone:] == E.HIT).all() and (out[gone:] == pages[gone:]).all(), cycle
        if pshift <= 17:
            out, st = eng.get_small(u[gone:], l[gone:])
            assert (st == E.HIT).all() and (out == pages[gone:]).all(), cycle
        if fl:
            fps1, ok1 = eng.read_fingerprints(u[gone:], l[gone:])
            assert (ok0 == ok1).all() and (fps0 == fps1).all(), cycle
        if flags == "VERIFY":
            _, _, bad, _ = eng.verify_store()
            assert bad == 0, cycle
        eng.close()


def test_host_tier_retire_scratch_grows_across_laps(E, gpu):
    """Two demotions that lap the ring, the second retiring more records than the first, then a
    promotion of the newest records back to the arena."""
    bs, n = 4096, 140
    pages = np.stack([datagen.make_page("R", bs, 700 + i) for i in range(n)])     # ~62 records per lap
    for cycle in range(CYCLES):
        eng = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128,
                       host_tier_bytes=256 << 10)
        u = np.full(n, 6, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        assert eng.demote(u[:60], l[:60]) == 60
        assert eng.host_tier_stats()["retired_records"] == 0
        assert eng.demote(u[60:80], l[60:80]) == 20
        r1 = eng.host_tier_stats()["retired_records"]
        assert eng.demote(u[80:], l[80:]) == 60
        r2 = eng.host_tier_stats()["retired_records"]
        assert 0 < r1 < r2 - r1, (cycle, r1, r2)
        out, st = eng.get(u, l)
        hit = st == E.HIT
        assert ((st == E.HIT) | (st == E.MISS)).all() and hit[80:].all() and (out[hit] == pages[hit]).all(), cycle
        assert eng.entries() == int(hit.sum()) == n - r2, cycle
        assert eng.promote(u[80:], l[80:]) == 60
        assert eng.host_tier_stats()["promoted_records"] == 60
        out, st = eng.get_small(u[80:], l[80:])
        assert (st == E.HIT).all() and (out == pages[80:]).all(), cycle
        eng.close()


def test_import_and_page_move_scratch_grows(E, gpu):
    """Record imports and page moves of increasing size on an engine without a host tier."""
    from edge_fuse_b200 import sharding
    bs = 4096
    src_pages = _pages(bs, 64, 300)
    for cycle in range(CYCLES):
        eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
        held = []
        for first, k in ((0, 10), (100, 100)):
            rows = sharding.pack_records(np.full(k, 7), np.arange(first, first + k), np.arange(k) + 10, 1,
                                         np.full(k, 100))
            d_rows = eng.dev_alloc(rows.nbytes)
            held.append(d_rows)
            eng.h2d(d_rows, rows)
            eng.import_records_dev(k, d_rows, 0)
        eng.sync()
        keys = np.concatenate([np.arange(10), np.arange(100, 200)]).astype(np.uint64)
        status, owner = eng.locate(np.full(len(keys), 7, dtype=np.uint64), keys)
        assert (status == E.REMOTE).all() and (owner == 1).all() and eng.stats()["remote_entries"] == 110, cycle
        src, dst = eng.dev_alloc(64 * bs), eng.dev_alloc(64 * bs)
        held += [src, dst]
        eng.h2d(src, src_pages)
        for m in (8, 64):
            dst_idx = np.arange(m)[::-1].copy()
            src_idx = (np.arange(m) * 5) % m
            eng.move_pages(m, dst, src, dst_idx=dst_idx, src_idx=src_idx)
            got = np.zeros((64, bs), dtype=np.uint8)
            eng.d2h(got, dst)
            assert (got[dst_idx] == src_pages[src_idx]).all(), (cycle, m)
        for p in held:
            eng.dev_free(p)
        eng.close()


def test_snapshot_then_load_into_a_fresh_engine(E, gpu, tmp_path):
    bs, n = 65536, 100
    pages = _pages(bs, n, 900)
    for cycle in range(CYCLES):
        path = str(tmp_path / f"c{cycle}.snap")
        eng = E.Engine(pshift=16, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.FINGERPRINT)
        u = np.full(n, 31, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        fps, _ = eng.read_fingerprints(u, l)
        assert E.snapshot_finish(eng.snapshot_begin(path)) == n
        eng.close()
        fresh = E.Engine(pshift=16, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.FINGERPRINT)
        assert fresh.load(path) == n
        out, st = fresh.get(u, l)
        assert (st == E.HIT).all() and (out == pages).all(), cycle
        assert (fresh.read_fingerprints(u, l)[0] == fps).all(), cycle
        fresh.close()
