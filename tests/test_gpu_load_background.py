"""GPU tests of background loads (cmb200_load_open / _step / _close, CMB200_LOAD=background).

Without other calls, a stepped load leaves what cmb200_load_chain leaves, and the chain goes on.  With
calls between the steps, every get returns the page of the "as-if store" (the whole file loaded at open,
then every call since) or a miss, never a page of the file that a later call superseded."""
import os
import random
import threading

import numpy as np
import pytest

import datagen
import key_edges
import load_model as LM
import snapshot_chain as sc
import store_machine as SM

pytestmark = pytest.mark.gpu

NH = 9


def _pages(bs, n, seed):
    kinds = "RTZMPAXS"
    return np.stack([datagen.make_page(kinds[(seed + i) % 8], bs, seed * 131 + i) for i in range(n)])


def _arr(addrs):
    return (np.array([a[0] for a in addrs], dtype=np.uint64), np.array([a[1] for a in addrs], dtype=np.uint64))


class _Writer:
    """Engines that write a chain, and the pages they hold by address."""

    def __init__(self, E, oracle, engines, pshift):
        self.E, self.O, self.engines, self.bs = E, oracle, engines, 1 << pshift
        self.ts = 1
        self.pages = {}

    def _own(self, addrs):
        g = len(self.engines)
        out = [[] for _ in range(g)]
        for i, a in enumerate(addrs):
            out[self.E.owner(self.O.addr_key(*a), g)].append(i)
        return out

    def put(self, addrs, pages):
        ts = np.arange(self.ts, self.ts + len(addrs), dtype=np.uint64)
        self.ts += len(addrs)
        for e, idx in zip(self.engines, self._own(addrs)):
            if idx:
                u, l = _arr([addrs[i] for i in idx])
                e.put(u, l, pages[idx], ts=ts[idx])
        for a, p in zip(addrs, pages):
            self.pages[a] = bytes(p)

    def unset(self, addrs):
        for e, idx in zip(self.engines, self._own(addrs)):
            if idx:
                e.unset(*_arr([addrs[i] for i in idx]))
        for a in addrs:
            self.pages.pop(a, None)

    def tick(self, base, delta):
        self.E.snapshot_finish(self.E.chain_begin([e.h for e in self.engines], base, delta))


def _write_chain(E, oracle, base, geo, pshift, n, deltas, g=1):
    engines = [E.Engine(**geo) for _ in range(g)]
    w = _Writer(E, oracle, engines, pshift)
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(n)]
    w.put(pool, _pages(w.bs, n, 1))
    w.tick(base, False)
    rnd = random.Random(pshift * 10 + deltas)
    for t in range(deltas):
        put = rnd.sample(pool, n // 5)
        w.put(put, _pages(w.bs, len(put), 10 + t))
        w.unset(rnd.sample(pool, n // 10))
        w.tick(base, True)
    for e in engines:
        e.close()
    return pool, w.pages


def _state(E, engines, pool, path):
    """Everything a load leaves, engine by engine: records, fingerprints, checkpoint words (the tag, which
    names the arena offset, left out), entries, and the store as a saved file reads back (with ts)."""
    g = len(engines)
    out = []
    for e in engines:
        u, l = _arr(pool)
        words, ok = e.read_checkpoints(u, l)
        fps, fok = e.read_fingerprints(u, l)
        out.append((e.read_records(u, l), fps.tolist(), fok.tolist(), words[:, 1:].tolist(), ok.tolist(), e.entries()))
    E.save_set([e.h for e in engines], path)
    saved, _ = sc.replay_chain(path)
    return out, {a: (r[0], r[1], r[2], r[3]) for a, r in saved.items()}, g


def _no_traffic_params():
    out = []
    for pshift in (12, 16, 17):
        for g in (1, 2):
            for tier in (False, True):
                out.append(pytest.param(pshift, g, tier, id=f"p{pshift}-g{g}-{'tier' if tier else 'hbm'}"))
    return out


@pytest.mark.parametrize("pshift,g,tier", _no_traffic_params())
def test_a_stepped_load_leaves_what_load_chain_leaves(E, gpu, oracle, tmp_path, pshift, g, tier):
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=(96 if tier else 256) << 20, max_batch=16,
               flags=E.FINGERPRINT)
    n = {12: 160, 16: 100, 17: 60}[pshift]
    if tier:
        geo["arena_bytes"] = max(n * (1 << pshift) // 3, 8 << 20)
    tier_bytes = (256 << 20) if tier else 0
    for deltas in (0, 3):
        base = str(tmp_path / f"d{deltas}" / "cachemap_b200.snap")
        os.makedirs(os.path.dirname(base))
        pool, _ = _write_chain(E, oracle, base, dict(geo, arena_bytes=256 << 20), pshift, n, deltas, g)
        ref = [E.Engine(host_tier_bytes=tier_bytes, **geo) for _ in range(g)]
        want_n = E.load_chain([e.h for e in ref], base)
        want = _state(E, ref, pool, str(tmp_path / "ref.snap"))
        for e in ref:
            e.close()
        for step in (1, 0, 7):          # 7 last: it ticks the chain on
            got_e = [E.Engine(host_tier_bytes=tier_bytes, **geo) for _ in range(g)]
            ld = E.Loader([e.h for e in got_e], base)
            assert ld.total >= want_n[0]
            steps = 0
            while ld.step(step):
                steps += 1
            assert ld.close() == want_n
            assert _state(E, got_e, pool, str(tmp_path / "got.snap")) == want, (deltas, step)
            if step == 7 and not tier:
                # the chain goes on from the stepped load: the next delta, loaded with its chain, is the store
                w = _Writer(E, oracle, got_e, pshift)
                extra = [oracle.addr_compose((n + i) << pshift, NH, 0, pshift) for i in range(5)]
                w.put(extra, _pages(w.bs, 5, 77))
                w.tick(base, True)
                again = [E.Engine(**geo) for _ in range(g)]
                assert E.load_chain([e.h for e in again], base)[1] == deltas + 1
                assert _state(E, again, pool + extra, str(tmp_path / "a.snap"))[1] == \
                    _state(E, got_e, pool + extra, str(tmp_path / "b.snap"))[1]
                for e in again:
                    e.close()
            for e in got_e:
                e.close()


# ---- conflicts: calls between the steps ----------------------------------------------------------

class _AsIf:
    """The as-if store: the file's pages, then every call since, by address; one record per store key."""

    def __init__(self, oracle, pages):
        self.O = oracle
        self.pages = dict(pages)

    def _drop_key(self, a):
        k = self.O.addr_key(*a)
        for b in [b for b in self.pages if self.O.addr_key(*b) == k]:
            del self.pages[b]

    def put(self, a, page):
        self._drop_key(a)
        self.pages[a] = bytes(page)

    def unset(self, a):
        self._drop_key(a)

    def invalidate(self, u, lo, hi):
        for b in [b for b in self.pages if b[0] == u and lo <= b[1] <= hi]:
            del self.pages[b]

    def rename(self, uf, ut, lo, hi):
        moved = {(ut, b[1]): p for b, p in self.pages.items() if b[0] == uf and lo <= b[1] <= hi}
        self.invalidate(uf, lo, hi)
        for a, p in moved.items():
            self.put(a, p)

    def check(self, E, eng, addrs):
        """Every get of eng (both get paths) is the as-if page or a miss -> hits."""
        u, l = _arr(addrs)
        hits = 0
        for fn in (eng.get, eng.get_small):
            out, st = fn(u, l)
            for i, a in enumerate(addrs):
                if st[i] == E.HIT:
                    assert a in self.pages and bytes(out[i]) == self.pages[a], (fn.__name__, a)
                    hits += 1
                else:
                    assert st[i] in (E.MISS, E.BAD_ENTRY), (a, st[i])
        return hits


def _conflict_setup(E, oracle, tmp_path, extra_addrs=(), host_tier=0, arena=64 << 20):
    pshift = 12
    geo = dict(pshift=pshift, accel=12, capacity=4096, arena_bytes=arena, max_batch=16, flags=E.FINGERPRINT)
    base = str(tmp_path / "cachemap_b200.snap")
    w = _Writer(E, oracle, [E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=16,
                                     flags=E.FINGERPRINT)], pshift)
    pool = [oracle.addr_compose(i << pshift, NH, 0, pshift) for i in range(96)] + list(extra_addrs)
    w.put(pool, _pages(4096, len(pool), 3))
    w.tick(base, False)
    w.engines[0].close()
    eng = E.Engine(host_tier_bytes=host_tier, **geo)
    return eng, base, pool, _AsIf(oracle, w.pages)


def _key_group():
    fx = key_edges.load()
    return [tuple(a) for a in fx["groups"]["pair0"]]


@pytest.mark.parametrize("first", [0, 40])
def test_puts_win_over_the_file(E, gpu, oracle, tmp_path, first):
    y1, y2 = _key_group()
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, extra_addrs=[y1])
    ld = E.Loader([eng.h], base)
    if first:
        ld.step(first)
    p = _pages(4096, 3, 50)
    eng.put(*_arr([pool[80], pool[1]]), p[:2])           # one not loaded yet, one loaded
    asif.put(pool[80], p[0]); asif.put(pool[1], p[1])
    eng.put(*_arr([y2]), p[2:3])                           # shares its key with the file's y1
    asif.put(y2, p[2])
    asif.check(E, eng, pool + [y2])
    while ld.step(5):
        asif.check(E, eng, pool + [y2])
    ld.close()
    assert asif.check(E, eng, pool + [y2]) >= 2 * 96
    u, l = _arr([pool[80], y2])
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and bytes(out[0]) == bytes(p[0]) and bytes(out[1]) == bytes(p[2])


def test_unset_by_a_colliding_key_keeps_the_file_page_out(E, gpu, oracle, tmp_path):
    y1, y2 = _key_group()
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, extra_addrs=[y1])
    ld = E.Loader([eng.h], base)
    eng.unset(*_arr([y2]))
    asif.unset(y2)
    while ld.step(7):
        asif.check(E, eng, pool)
    ld.close()
    asif.check(E, eng, pool)
    _, st = eng.get(*_arr([y1]))
    assert st[0] != E.HIT


@pytest.mark.parametrize("span", ["keyed", "scan"])
def test_invalidate_keeps_the_file_pages_out(E, gpu, oracle, tmp_path, span):
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path)
    ld = E.Loader([eng.h], base)
    ld.step(20)
    hi = 60 if span == "keyed" else (1 << 44) - 1
    eng.invalidate(NH, 10, hi)
    asif.invalidate(NH, 10, hi)
    while ld.step(9):
        asif.check(E, eng, pool)
    ld.close()
    assert asif.check(E, eng, pool) == 2 * len(asif.pages)


@pytest.mark.parametrize("first", [0, 48])
def test_rename_moves_or_drops_never_serves_the_old(E, gpu, oracle, tmp_path, first):
    dst = [oracle.addr_compose(i << 12, NH + 1, 0, 12) for i in range(96)]
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, extra_addrs=dst)
    ld = E.Loader([eng.h], base)
    if first:
        ld.step(first)
    eng.rename(NH, NH + 1, 0, 200)
    asif.rename(NH, NH + 1, 0, 200)
    while ld.step(11):
        asif.check(E, eng, pool)
    ld.close()
    asif.check(E, eng, pool)
    _, st = eng.get(*_arr(pool[:96]))
    assert (st != E.HIT).all()


def test_patches_hit_what_is_loaded_and_drop_what_is_not(E, gpu, oracle, tmp_path):
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path)
    ld = E.Loader([eng.h], base)
    ld.step(48)
    _, st0 = eng.get(*_arr(pool))
    loaded = [a for a, s in zip(pool, st0) if s == E.HIT]
    absent = [a for a, s in zip(pool, st0) if s != E.HIT]
    assert loaded and absent
    targets = [loaded[0], absent[0]]
    st = eng.patch(*_arr(targets), [100, 100], [b"patched!", b"patched!"])
    assert list(st) == [E.HIT, E.MISS]
    page = bytearray(asif.pages[loaded[0]])
    page[100:108] = b"patched!"
    asif.pages[loaded[0]] = bytes(page)
    asif.unset(absent[0])                                  # the as-if store held it: the patch makes it a miss at worst
    while ld.step(13):
        asif.check(E, eng, pool)
    ld.close()
    asif.check(E, eng, pool)
    _, st = eng.get(*_arr([absent[0]]))
    assert st[0] != E.HIT


def test_tier_laps_during_the_load(E, gpu, oracle, tmp_path):
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, host_tier=1 << 20, arena=4 << 20)
    ld = E.Loader([eng.h], base)
    more = [oracle.addr_compose(i << 12, NH + 2, 0, 12) for i in range(400)]
    p = _pages(4096, len(more), 9)
    k = 0
    while ld.step(8):
        # puts demoted at once: the tier of 1 MiB laps, retiring what it held, the file's pages included
        eng.put(*_arr(more[k:k + 40]), p[k:k + 40])
        eng.demote(*_arr(more[k:k + 40] + pool))
        for a, q in zip(more[k:k + 40], p[k:k + 40]):
            asif.put(a, q)
        k = (k + 40) % len(more)
        asif.check(E, eng, pool + more)
    ld.close()
    asif.check(E, eng, pool + more)
    assert eng.host_tier_stats()["retired_records"] > 0


def test_snapshots_are_refused_while_a_load_is_open(E, gpu, oracle, tmp_path):
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path)
    ld = E.Loader([eng.h], base)
    with pytest.raises(RuntimeError, match="load"):
        E.snapshot_begin([eng.h], str(tmp_path / "x.snap"))
    with pytest.raises(RuntimeError, match="load"):
        E.save_set([eng.h], str(tmp_path / "x.snap"))
    with pytest.raises(RuntimeError, match="open already"):
        E.Loader([eng.h], base)
    ld.step(0)
    ld.close()
    E.save_set([eng.h], str(tmp_path / "x.snap"))


def test_small_gets_during_a_load_return_whole_pages(E, gpu, oracle, tmp_path):
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path)
    ld = E.Loader([eng.h], base)
    stop = threading.Event()
    bad = []

    def reader():
        u, l = _arr(pool)
        while not stop.is_set():
            out, st = eng.get_small(u, l)
            for i, a in enumerate(pool):
                if st[i] == E.HIT and bytes(out[i]) != asif.pages[a]:
                    bad.append(a)

    th = threading.Thread(target=reader)
    th.start()
    try:
        while ld.step(3):
            pass
    finally:
        stop.set()
        th.join()
    ld.close()
    assert not bad
    assert asif.check(E, eng, pool) == 2 * len(pool)


def test_a_load_with_traffic_leaves_no_chain_state(E, gpu, oracle, tmp_path):
    pshift = 12
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=16, flags=E.FINGERPRINT)
    base = str(tmp_path / "cachemap_b200.snap")
    pool, _ = _write_chain(E, oracle, base, geo, pshift, 64, 2)
    quiet = E.Engine(**geo)
    ld = E.Loader([quiet.h], base)
    while ld.step(10):
        pass
    ld.close()
    E.snapshot_finish(E.chain_begin([quiet.h], base, True))          # a quiet load continues the chain
    busy = E.Engine(**geo)
    ld = E.Loader([busy.h], base)
    ld.step(10)
    busy.put(*_arr([pool[60]]), _pages(4096, 1, 99))
    while ld.step(10):
        pass
    ld.close()
    with pytest.raises(RuntimeError):
        E.chain_begin([busy.h], base, True)
    E.snapshot_finish(E.chain_begin([busy.h], base, False))
    quiet.close()
    busy.close()


def _file_reads(cm, model, bs):
    """{(nh, page): page bytes} of every page of the model that the map answers; each answer is checked."""
    got = {}
    for nh, data in model.items():
        n = len(data) // bs
        off = np.arange(n, dtype=np.uint64) * np.uint64(bs)
        out, hit = cm.get_batch(off, np.full(n, nh, dtype=np.uint64), np.ones(n, dtype=np.uint32))
        for p in np.nonzero(hit)[0]:
            assert out[p].tobytes() == bytes(data[p * bs:(p + 1) * bs]), (nh, int(p))
            got[(nh, int(p))] = True
    return got


def test_drop_in_restart_over_two_engines_in_the_background(E, gpu, tmp_path, monkeypatch):
    d = str(tmp_path / "cache")
    os.makedirs(d)
    for k in ("CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("CMB200_DEVICES", "0,0")
    monkeypatch.setenv("CMB200_ARENA_MB", "512")
    # 60 000 pages: the loader thread takes 4 096 records per step, so the load runs many steps
    bs, n = 4096, 60000
    rng = np.random.default_rng(5)
    files = {}
    for nh in (21, 22, 23):
        data = rng.integers(0, 16, size=bs * n // 3, dtype=np.uint8)
        data[::2] = 0x41
        files[nh] = bytearray(data.tobytes())
    cm = E.Cachemap(d, 1 << 17, 12, 12)
    for nh, data in files.items():
        cm.pwrite(nh, 1, 0, bytes(data))
    cm.free()
    monkeypatch.setenv("CMB200_LOAD", "background")
    cm = E.Cachemap(d, 1 << 17, 12, 12)
    model = {nh: bytearray(b) for nh, b in files.items()}
    cm.pwrite(21, 1, 5000, b"x" * 9000)                   # partial pages patch, whole pages put
    model[21][5000:14000] = b"x" * 9000
    cm.invalidate(22, 1, 8192, 3 * bs)
    gone = {(22, p) for p in range(2, 5)}
    cm.rename(23, 24, 1)
    model[24] = model.pop(23)
    loading, _, total = cm.load_progress()
    assert loading, "the load ended before the writes, the invalidation and the rename were made"
    assert total == n
    while cm.load_progress()[0]:
        pass
    got = _file_reads(cm, model, bs)
    assert not gone & set(got)
    # what the load met no change for is all there; moved and written pages hit or miss, never stale
    assert {(22, p) for p in range(n // 3)} - gone <= set(got)
    assert cm.checkpoint() == 0
    cm.free()
    monkeypatch.delenv("CMB200_LOAD")
    cm = E.Cachemap(d, 1 << 17, 12, 12)
    again = _file_reads(cm, model, bs)
    assert set(again) == set(got)
    cm.free()


def test_a_lapped_put_over_an_unloaded_file_page_stays_a_miss(E, gpu, oracle, tmp_path):
    """A page put during the load over a file address not loaded yet, then retired by a host-tier lap, and
    its tombstone dropped by a table rebuild: the file's older page must not come back."""
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, host_tier=256 << 10, arena=16 << 20)
    ld = E.Loader([eng.h], base)
    target = pool[90]
    eng.put(*_arr([target]), _pages(4096, 1, 61))
    asif.put(target, _pages(4096, 1, 61)[0])
    eng.demote(*_arr([target]))
    more = [oracle.addr_compose(i << 12, NH + 3, 0, 12) for i in range(160)]
    noise = np.random.default_rng(62).integers(0, 256, size=(len(more), 4096), dtype=np.uint8)
    eng.put(*_arr(more), noise)                           # 640 KiB that does not compress: demoted, it laps the tier
    eng.demote(*_arr(more))
    for a, q in zip(more, noise):
        asif.put(a, q)
    _, st = eng.get(*_arr([target]))
    assert st[0] != E.HIT and eng.host_tier_stats()["retired_records"] > 0
    # more tombstones than table_slots / 8, then a compaction: the table is rebuilt without them
    purge = [(NH + 4, l) for l in range(eng.stats()["table_slots"] // 8 + 64)]
    eng.put(*_arr(purge), _pages(4096, 8, 63)[np.arange(len(purge)) % 8])
    eng.unset(*_arr(purge))
    eng.compact()
    assert eng.stats()["tombstones"] == 0
    while ld.step(16):
        asif.check(E, eng, pool + more)
    ld.close()
    asif.check(E, eng, pool + more)
    _, st = eng.get(*_arr([target]))
    assert st[0] != E.HIT


def test_puts_of_fenced_addresses_win(E, gpu, oracle, tmp_path):
    """Addresses invalidated, unset or renamed before the load reached them, then put again: the new page
    is served, neither the file's nor a miss."""
    dst = [oracle.addr_compose(i << 12, NH + 1, 0, 12) for i in range(8)]
    eng, base, pool, asif = _conflict_setup(E, oracle, tmp_path, extra_addrs=dst)
    ld = E.Loader([eng.h], base)
    eng.invalidate(NH, 70, 79)
    asif.invalidate(NH, 70, 79)
    eng.unset(*_arr(pool[80:84]))
    for a in pool[80:84]:
        asif.unset(a)
    eng.rename(NH, NH + 1, 0, 7)
    asif.rename(NH, NH + 1, 0, 7)
    again = pool[70:74] + pool[80:82] + pool[0:2] + dst[0:2]
    p = _pages(4096, len(again), 64)
    eng.put(*_arr(again), p)
    for a, q in zip(again, p):
        asif.put(a, q)
    while ld.step(9):
        asif.check(E, eng, pool)
    ld.close()
    asif.check(E, eng, pool)
    out, st = eng.get(*_arr(again))
    assert (st == E.HIT).all() and all(bytes(out[i]) == bytes(p[i]) for i in range(len(again)))


# ---- seeded interleavings of load steps with every store operation (tests/load_model.py) -------------

def _run_load_machine(E, oracle, cfg, seed, tmp_path):
    key_of = lambda a: oracle.addr_key(*a)      # noqa: E731
    U = list(dict.fromkeys(SM.universe(cfg)))
    geo = dict(pshift=cfg.pshift, accel=cfg.accel, max_batch=cfg.max_batch, flags=cfg.flags)
    writer = E.Engine(capacity=cfg.load_slots // 4, arena_bytes=cfg.load_arena, table_slots=cfg.load_slots, **geo)
    rows = [(u, l) for u in cfg.us for l in range(cfg.nl)] + SM.edge_addrs()
    specs = [(SM.KINDS[i % len(SM.KINDS)], seed * 10_000 + i) for i in range(len(rows))]
    writer.put(*_arr(rows), SM.pages_of(cfg, specs))
    base = str(tmp_path / "cachemap_b200.snap")
    E.snapshot_finish(E.chain_begin([writer.h], base, False))
    writer.put(*_arr(rows[::5]), SM.pages_of(cfg, [("T", seed * 10_000 + 5000 + i) for i in range(len(rows[::5]))]))
    writer.unset(*_arr(rows[3::11]))
    E.snapshot_finish(E.chain_begin([writer.h], base, True))
    out, st = writer.get(*_arr(U))
    writer.close()
    model = LM.AsIfModel(key_of, {a: out[i].tobytes() for i, a in enumerate(U) if st[i] == E.HIT})
    eng = E.Engine(capacity=cfg.table_slots // 4, arena_bytes=cfg.arena_bytes, table_slots=cfg.table_slots,
                   host_tier_bytes=cfg.tier_bytes, **geo)
    ld = E.Loader([eng.h], base)
    loading, log = True, []
    for i, op in enumerate(LM.gen_load_ops(cfg, seed)):
        kind = op[0]
        log.append(f"{i:4d} {op[0]} {op[1] if kind in ('step',) else ''}")
        if kind == "step":
            loading = loading and ld.step(op[1])
        elif kind in ("put", "put_async"):
            _, addrs, sp, ts, valid = op
            pages = SM.pages_of(cfg, sp)
            lens = eng.put(*_arr(addrs), pages, ts=None if ts is None else np.array(ts, dtype=np.uint64),
                           valid=None if valid is None else np.array(valid, dtype=np.uint8))
            model.put(addrs, pages, valid, lens)
        elif kind == "unset":
            eng.unset(*_arr(op[1]))
            model.unset(op[1])
        elif kind == "invalidate":
            eng.invalidate(op[1], op[2], op[3])
            model.invalidate(op[1], op[2], op[3])
        elif kind == "rename":
            _, dropped = eng.rename(op[1], op[2], op[3], op[4])
            if op[1] != op[2]:
                model.rename(op[1], op[2], op[3], op[4], dropped)
        elif kind == "patch":
            _, addrs, spans, ts = op
            status = eng.patch(*_arr(addrs), [s[0] for s in spans], [SM.span_bytes(s) for s in spans],
                               ts=None if ts is None else np.array(ts, dtype=np.uint64))
            model.patch(addrs, spans, status)
        elif kind == "demote":
            eng.demote(*_arr(op[1]))
        elif kind == "promote":
            eng.promote(*_arr(op[1]))
        elif kind == "compact":
            eng.compact()
        elif kind == "verify_store":
            eng.verify_store()
        for fn in (eng.get, eng.get_small):
            pages, status = fn(*_arr(U))
            bad = model.check(U, status, pages)
            assert bad is None, (f"config {cfg.name} seed {seed} op {i} ({kind}, {fn.__name__}): {bad}\n"
                                 + "\n".join(log[-30:]))
    while loading and ld.step(0):
        pass
    records, _ = ld.close()
    assert records > 0
    for fn in (eng.get, eng.get_small):
        pages, status = fn(*_arr(U))
        assert model.check(U, status, pages) is None
    eng.close()


@pytest.mark.parametrize("name,seed", [("A", 11), ("C", 31), ("D", 41), ("E", 51)])
def test_seeded_interleavings_of_load_steps_and_store_operations(E, gpu, oracle, tmp_path, monkeypatch, name, seed):
    cfg = SM.CONFIGS[name]
    for k, v in cfg.environ().items():
        monkeypatch.setenv(k, v)
    _run_load_machine(E, oracle, cfg, seed, tmp_path)
