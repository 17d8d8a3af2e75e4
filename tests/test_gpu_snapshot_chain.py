"""GPU tests of snapshot chains (cmb200_chain_begin / cmb200_load_chain): after every tick the base plus
its deltas load into a fresh engine as the store of that tick; a delta holds exactly the keys put since
the last tick and the addresses that stopped being live, and nothing for records that only moved; damaged
chains load up to their valid prefix; the drop-in keeps a chain with CMB200_CHECKPOINT_DELTAS."""
import os
import random
import shutil
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import datagen
import key_edges
import snapshot_chain as sc

pytestmark = pytest.mark.gpu

NH = 5


def _tick(E, engines, base, delta):
    """One chain tick over the engines -> the file it wrote (records as snapshot_finish reports them)."""
    s = E.chain_begin([e.h for e in engines], base, delta)
    E.snapshot_finish(s)
    if not delta:
        return base, None
    k = max(int(n.rsplit(".d", 1)[1]) for n in os.listdir(os.path.dirname(base))
            if n.startswith(os.path.basename(base) + ".d") and n.rsplit(".d", 1)[1].isdigit())
    return f"{base}.d{k}", sc.read_delta(f"{base}.d{k}")


class _Store:
    """Engines and the oracle's StoreModel, changed together; addresses are (u, l) pairs."""

    def __init__(self, E, oracle, engines, pshift, accel):
        self.E, self.O, self.engines, self.pshift = E, oracle, engines, pshift
        self.model = oracle.StoreModel(pshift, accel)
        self.ts = 1

    def _by_engine(self, addrs):
        g = len(self.engines)
        out = [[] for _ in range(g)]
        for i, a in enumerate(addrs):
            out[self.E.owner(self.O.addr_key(*a), g)].append(i)
        return out

    def put(self, addrs, pages):
        ts = np.arange(self.ts, self.ts + len(addrs), dtype=np.uint64)
        self.ts += len(addrs)
        for e, idx in zip(self.engines, self._by_engine(addrs)):
            if idx:
                e.put(np.array([addrs[i][0] for i in idx], dtype=np.uint64),
                      np.array([addrs[i][1] for i in idx], dtype=np.uint64), pages[idx], ts=ts[idx])
        for a, p in zip(addrs, pages):
            self.model.put(*key_edges.cachemap_args(a[0], a[1], self.pshift), p)

    def unset(self, addrs):
        for e, idx in zip(self.engines, self._by_engine(addrs)):
            if idx:
                e.unset(np.array([addrs[i][0] for i in idx], dtype=np.uint64),
                        np.array([addrs[i][1] for i in idx], dtype=np.uint64))
        for a in addrs:
            self.model.unset(*a)

    def live(self):
        """{(u, l): record bytes} of the model."""
        return {r[0]: self.O.record_prefix(r[0][0], r[0][1], r[1]) + r[2] for r in self.model.rec.values()}


def _pool(oracle, pshift, n):
    fx = key_edges.load()
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(n)]
    for g in fx["groups"].values():
        pool += list(g)
    return pool


def _agrees(E, eng, store, pool, model):
    """eng answers every address of the pool as `model` (a StoreModel) does."""
    u = np.array([a[0] for a in pool], dtype=np.uint64)
    l = np.array([a[1] for a in pool], dtype=np.uint64)
    want = {"hit": E.HIT, "miss": E.MISS, "bad entry": E.BAD_ENTRY}
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        for i, a in enumerate(pool):
            s, page = model.get_status(*key_edges.cachemap_args(a[0], a[1], store.pshift))
            assert st[i] == want[s], (i, a, st[i], s)
            if s == "hit":
                assert bytes(out[i]) == bytes(page)
    assert eng.entries() == model.entries()


def _replayed(base):
    state, k = sc.replay_chain(base)
    return {a: r[3] for a, r in state.items()}, k


def _pages(bs, n, seed):
    kinds = "RTZMPAXS"
    return np.stack([datagen.make_page(kinds[(seed + i) % 8], bs, seed * 131 + i) for i in range(n)])


@pytest.mark.parametrize("pshift", [12, 16])
def test_every_tick_loads_as_the_store_of_that_tick(E, gpu, oracle, tmp_path, pshift):
    import copy
    bs = 1 << pshift
    geo = dict(pshift=pshift, accel=12, capacity=4096, arena_bytes=256 << 20, max_batch=64, flags=E.FINGERPRINT)
    eng = E.Engine(host_tier_bytes=64 << 20, **geo)
    s = _Store(E, oracle, [eng], pshift, 12)
    pool = _pool(oracle, pshift, 80)
    rnd = random.Random(pshift)
    base = str(tmp_path / "cachemap_b200.snap")
    s.put(pool[:60], _pages(bs, 60, 1))
    _tick(E, [eng], base, False)
    for t in range(5):
        live_before = set(s.live())
        put = rnd.sample(pool, rnd.randrange(1, 25))
        s.put(put, _pages(bs, len(put), 10 + t))
        gone = rnd.sample(pool, rnd.randrange(0, 12))
        s.unset(gone)
        if t == 2:       # a tier round between two ticks: records move, nothing changes
            u = np.array([a[0] for a in pool[:30]], dtype=np.uint64)
            l = np.array([a[1] for a in pool[:30]], dtype=np.uint64)
            eng.demote(u, l)
        path, d = _tick(E, [eng], base, True)
        live = s.live()
        keys_put = {oracle.addr_key(*a) for a in put}
        want_recs = {a for a in live if oracle.addr_key(*a) in keys_put}
        assert {sc.addr_of(r[3]) for r in d["records"]} == want_recs
        assert len(d["records"]) == len(want_recs)
        assert set(d["tombstones"]) == live_before - set(live)
        assert d["index"] == t + 1 and d["chain"] == sc.read_chain_id(base) != 0 and d["flags"] == 1
        assert _replayed(base) == (live, t + 1)
        e2 = E.Engine(**geo)
        assert E.load_chain([e2.h], base) == (len(live), t + 1)
        _agrees(E, e2, s, pool, copy.deepcopy(s.model))
        e2.close()
    eng.close()


def test_deltas_hold_what_changed_and_nothing_that_moved(E, gpu, oracle, tmp_path):
    pshift, bs, n = 12, 4096, 300
    geo = dict(pshift=pshift, accel=12, capacity=512, table_slots=1024, arena_bytes=64 << 20, max_batch=64,
               flags=E.FINGERPRINT)
    eng = E.Engine(host_tier_bytes=32 << 20, **geo)
    s = _Store(E, oracle, [eng], pshift, 12)
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(n)]
    base = str(tmp_path / "b.snap")
    s.put(pool, _pages(bs, n, 3))
    _tick(E, [eng], base, False)
    _, d = _tick(E, [eng], base, True)                   # nothing changed
    assert d["records"] == [] and d["tombstones"] == []
    s.unset(pool[100:300])                               # d = 200 unsets, m = 7 rewrites
    s.put(pool[:7], _pages(bs, 7, 4))
    _, d = _tick(E, [eng], base, True)
    assert len(d["records"]) == 7 and len(d["tombstones"]) == 200
    # demotion, promotion, compaction and the table rebuild it triggers (200 tombstones > 1024 / 8)
    u = np.array([a[0] for a in pool[:100]], dtype=np.uint64)
    l = np.array([a[1] for a in pool[:100]], dtype=np.uint64)
    assert eng.demote(u[:60], l[:60]) == 60
    assert eng.promote(u[:20], l[:20]) == 20
    assert eng.stats()["tombstones"] > 0
    eng.compact()
    assert eng.stats()["tombstones"] == 0
    _, d = _tick(E, [eng], base, True)
    assert d["records"] == [] and d["tombstones"] == []
    assert _replayed(base) == (s.live(), 3)
    # the fingerprint flag survives, and a verifying engine checks the loaded records
    e2 = E.Engine(**dict(geo, flags=E.VERIFY))
    assert E.load_chain([e2.h], base) == (100, 3)
    _, _, n_bad, checked = e2.verify_store()
    assert n_bad == 0 and checked == 100
    out, st = e2.get_small(u, l)
    assert (st == E.HIT).all() and e2.verify_stats()["verified"] == 100
    e2.close()
    eng.close()


def test_chain_moves_between_engine_counts(E, gpu, oracle, tmp_path):
    pshift, bs = 12, 4096
    geo = dict(pshift=pshift, accel=12, capacity=2048, arena_bytes=64 << 20, max_batch=64, device=0)
    pool = _pool(oracle, pshift, 200)
    for g_write, g_read in ((2, 1), (1, 2)):
        engs = [E.Engine(**geo) for _ in range(g_write)]
        s = _Store(E, oracle, engs, pshift, 12)
        base = str(tmp_path / f"g{g_write}.snap")
        s.put(pool[:150], _pages(bs, 150, 5))
        _tick(E, engs, base, False)
        s.put(pool[100:], _pages(bs, len(pool) - 100, 6))
        s.unset(pool[:20])
        _tick(E, engs, base, True)
        readers = [E.Engine(**geo) for _ in range(g_read)]
        assert E.load_chain([e.h for e in readers], base) == (len(s.live()), 1)
        r = _Store(E, oracle, readers, pshift, 12)
        r.model = s.model
        for i, e in enumerate(readers):
            sub = [a for a in pool if E.owner(oracle.addr_key(*a), g_read) == i]
            out, st = e.get(np.array([a[0] for a in sub], dtype=np.uint64), np.array([a[1] for a in sub], dtype=np.uint64))
            for j, a in enumerate(sub):
                want, page = s.model.get_status(*key_edges.cachemap_args(a[0], a[1], pshift))
                assert st[j] == {"hit": E.HIT, "miss": E.MISS, "bad entry": E.BAD_ENTRY}[want]
                if want == "hit":
                    assert bytes(out[j]) == bytes(page)
        # the readers continue the chain
        r.put(pool[:5], _pages(bs, 5, 7))
        path, d = _tick(E, readers, base, True)
        assert path.endswith(".d2") and len(d["records"]) == 5
        for e in engs + readers:
            e.close()


def test_puts_during_a_delta_write_are_not_in_it(E, gpu, oracle, tmp_path):
    pshift, bs = 16, 65536
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=256 << 20, max_batch=64)
    eng = E.Engine(**geo)
    s = _Store(E, oracle, [eng], pshift, 12)
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(200)]
    base = str(tmp_path / "live.snap")
    s.put(pool[:100], _pages(bs, 100, 8))
    _tick(E, [eng], base, False)
    s.put(pool[50:150], _pages(bs, 100, 9))
    at_begin = s.live()
    h = E.chain_begin([eng.h], base, True)
    s.put(pool[140:200], _pages(bs, 60, 10))
    s.unset(pool[:30])
    s.put(pool[60:70], _pages(bs, 10, 11))
    eng.compact()
    assert E.snapshot_finish(h) == 100
    assert _replayed(base) == (at_begin, 1)
    _, d = _tick(E, [eng], base, True)
    assert len(d["tombstones"]) == 30 and len(d["records"]) == 70
    assert _replayed(base) == (s.live(), 2)
    eng.close()


def _write_chain(E, oracle, tmp_path, name, ticks=4):
    """A base and `ticks` deltas -> (base path, geometry, [store of tick 0 .. ticks], pool)."""
    import copy
    pshift, bs = 12, 4096
    geo = dict(pshift=pshift, accel=12, capacity=2048, arena_bytes=64 << 20, max_batch=64)
    eng = E.Engine(**geo)
    s = _Store(E, oracle, [eng], pshift, 12)
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(300)]
    d = tmp_path / name
    d.mkdir()
    base = str(d / "cachemap_b200.snap")
    s.put(pool[:200], _pages(bs, 200, 12))
    _tick(E, [eng], base, False)
    hist = [copy.deepcopy(s.model)]
    for t in range(ticks):
        s.put(pool[40 * t: 40 * t + 60], _pages(bs, 60, 13 + t))
        s.unset(pool[40 * t + 200: 40 * t + 210] + pool[t * 5: t * 5 + 3])
        _tick(E, [eng], base, True)
        hist.append(copy.deepcopy(s.model))
    eng.close()
    return base, geo, hist, pool, s


@pytest.mark.parametrize("shape", ["tmp_left", "d2_missing", "last_truncated", "foreign_id"])
def test_damaged_chains_load_their_valid_prefix(E, gpu, oracle, tmp_path, shape):
    base, geo, hist, pool, s = _write_chain(E, oracle, tmp_path, shape)
    if shape == "tmp_left":
        open(base + ".d5.tmp", "wb").write(b"half a delta")
        want = 4
    elif shape == "d2_missing":
        os.remove(base + ".d2")
        want = 1
    elif shape == "last_truncated":
        raw = open(base + ".d4", "rb").read()
        open(base + ".d4", "wb").write(raw[:-7])
        want = 3
    else:
        d = sc.read_delta(base + ".d3")
        sc.write_delta(base + ".d3", d["pshift"], d["chain"] ^ 1, 3, d["tombstones"], d["records"])
        want = 2
    e2 = E.Engine(**geo)
    assert E.load_chain([e2.h], base)[1] == want
    _agrees(E, e2, s, pool, hist[want])
    if shape == "tmp_left":             # a whole chain: the next tick continues it
        path, d = _tick(E, [e2], base, True)
        assert path.endswith(".d5") and d["records"] == [] and d["tombstones"] == []
    else:                               # the run ended early: the next tick must write a base
        with pytest.raises(RuntimeError):
            E.chain_begin([e2.h], base, True)
        _tick(E, [e2], base, False)
        assert sc.valid_deltas(base) == []
    e2.close()


def test_a_load_that_dropped_records_leaves_no_chain(E, gpu, oracle, tmp_path):
    base, geo, hist, pool, s = _write_chain(E, oracle, tmp_path, "drop", ticks=2)
    small = E.Engine(**dict(geo, arena_bytes=1 << 18))
    n, k = E.load_chain([small.h], base)
    assert k == 2 and small.entries() < hist[2].entries()
    with pytest.raises(RuntimeError):
        E.chain_begin([small.h], base, True)
    small.close()



DROP_IN = textwrap.dedent("""
    import os, shutil, sys, time
    sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
    sys.path.insert(0, sys.argv[1])
    import datagen
    import edge_fuse_b200 as E
    src, dst, phase = sys.argv[2], sys.argv[3], sys.argv[4]
    pages = [datagen.make_page("RTZMPAXS"[i % 8], 4096, 7000 + i) for i in range(400)]
    if phase == "write":
        cm = E.Cachemap(src, 4096, 12, 12)
        for r in range(5):
            for i in range(r * 80, r * 80 + 80):
                cm.put(i << 12, 9, 0, pages[(i * 7 + r) % 400])
            time.sleep(1.5)
        time.sleep(1.5)
        shutil.copytree(src, dst)   # the directory as a crash leaves it: cachemap_free never runs
        print("files", " ".join(sorted(os.listdir(dst))), flush=True)
        os._exit(0)
    cm = E.Cachemap(dst, 4096, 12, 12)
    bad = sum(bytes(cm.get(i << 12, 9, 0) or b"") != bytes(pages[(i * 7 + i // 80) % 400]) for i in range(400))
    print("bad", bad, flush=True)
    cm.free()
""")


def test_drop_in_chain_survives_a_crash(E, gpu, tmp_path):
    script = tmp_path / "drive.py"
    script.write_text(DROP_IN)
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_CHECKPOINT_SEC="1", CMB200_CHECKPOINT_DELTAS="4")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, dst = tmp_path / "cache", tmp_path / "copy"
    src.mkdir()
    w = subprocess.run([sys.executable, str(script), root, str(src), str(dst), "write"], capture_output=True,
                       text=True, timeout=300, env=env)
    assert w.returncode == 0 and "cachemap_b200.snap.d1" in w.stdout, w.stdout + w.stderr[-3000:]
    r = subprocess.run([sys.executable, str(script), root, str(src), str(dst), "read"], capture_output=True,
                       text=True, timeout=300, env=env)
    assert r.returncode == 0 and "bad 0" in r.stdout, r.stdout + r.stderr[-3000:]
    shutil.rmtree(dst)
