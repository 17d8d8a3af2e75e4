"""GPU tests of ghost entries (CMB200_GHOST) and of the hit curve through the drop-in (CMB200_GHOST=1).

Engine level: seeded sequences of puts, evictions, gets on every path, unsets, invalidations on both paths,
renames and patches; after every step the ghost table (cmb200_ghost_read) and the statistics equal
tests/ghost_model.py's GhostTable word for word.  The same sequence without the flag (evictions as unsets)
gives the same statuses and pages.  Host-tier laps stamp what they retire in tier order.  Then the curve at
twice the capacity through the drop-in, against a second run at that capacity."""
import random

import numpy as np
import pytest

import ghost_model as G

pytestmark = pytest.mark.gpu

CAP = 256                      # 256 ghost entries: 64 sets, buckets of 4 evictions


def _page(bsize, a, version):
    rng = np.random.default_rng((a[0] * 1000003 + a[1]) * 7 + version)
    p = np.repeat(rng.integers(0, 256, size=bsize // 64, dtype=np.uint8), 64)   # compressible
    p[:24] = np.frombuffer(np.array([a[0], a[1], version], dtype=np.uint64).tobytes(), dtype=np.uint8)
    return p


def _get(E, e, path, addrs, valid=None):
    u = np.array([a[0] for a in addrs], dtype=np.uint64)
    l = np.array([a[1] for a in addrs], dtype=np.uint64)
    if path == "small":
        return e.get_small(u, l)
    if path == "batch":
        return e.get(u, l, valid=valid)
    n = len(u)
    dev = E.lib().cmb200_dev_alloc(e.h, n * e.bsize)
    try:
        st = np.zeros(n, dtype=np.int32)
        addr = np.stack([u, l], axis=1).astype(np.uint64)
        v = None if valid is None else np.ascontiguousarray(valid, dtype=np.uint8)
        assert E.lib().cmb200_get_batch_dev(e.h, n, addr.ctypes.data, None if v is None else v.ctypes.data,
                                            dev, st.ctypes.data) == 0
        out = np.zeros((n, e.bsize), dtype=np.uint8)
        assert E.lib().cmb200_memcpy_d2h(e.h, out.ctypes.data, dev, n * e.bsize) == 0
        return out, st
    finally:
        E.lib().cmb200_dev_free(e.h, dev)


def _check(e, g):
    tab = e.ghost_read()
    want = g.words()
    bad = np.nonzero((tab != want).any(axis=1))[0]
    assert len(bad) == 0, (bad[:4], tab[bad[:4]], want[bad[:4]])
    st = e.ghost_stats()
    ms = g.stats()
    for k, v in ms.items():
        assert st[k] == v, (k, st[k], v)


def _sequence(E, pshift, ghost, seed, steps=60, wide=False):
    """Runs one seeded sequence on a fresh engine.  ghost: with the flag, evictions by cmb200_evict_batch and
    the table checked after every step; without, evictions by cmb200_unset_batch.  wide: a pool of 1 200
    addresses, more than four times the table, evicted 60 at a time, and gets that ask mostly for pages
    evicted long ago, so that sets fill (the oldest way goes) and ghosts refault after more evictions than the
    table has entries (`beyond`).  Returns every get's statuses and pages."""
    # wide: a key table that holds the whole pool (4 x CAP slots would not); the ghost table still has CAP entries
    e = E.Engine(pshift=pshift, capacity=CAP, arena_bytes=256 << 20, max_batch=64, table_slots=4096 if wide else 0,
                 flags=E.GHOST if ghost else 0)
    g = G.GhostTable(CAP)
    rng = random.Random(seed)
    bs = 1 << pshift
    store = {}                              # address -> the page stored there
    version = [0]
    answers = []
    span = 400 if wide else 40
    pool = [(u, l) for u in (11, 12, 13) for l in range(span)]
    gone = []                               # evicted addresses, oldest first

    def arrays(addrs):
        return (np.array([a[0] for a in addrs], dtype=np.uint64), np.array([a[1] for a in addrs], dtype=np.uint64))

    def put(addrs):
        version[0] += 1
        pages = np.stack([_page(bs, a, version[0]) for a in addrs])
        e.put(*arrays(addrs), pages)
        for a, p in zip(addrs, pages):
            store[a] = p

    try:
        put(pool if wide else pool[:60])
        for _step in range(steps):
            op = rng.choice(["put", "evict", "evict", "get", "get", "get", "unset", "inv", "inv_scan", "rename",
                             "patch"])
            if op == "put":
                put(rng.sample(pool, 60 if wide else 12))
            elif op == "evict":
                live = list(store)
                addrs = rng.sample(live, min(len(live), 60 if wide else 8)) + rng.sample(pool, 3)
                addrs.insert(2, addrs[0])                           # a repeat: one ghost
                rng.shuffle(addrs)
                removed = []
                for a in addrs:
                    if a in store:
                        removed.append(a)
                        del store[a]
                gone.extend(removed)
                if ghost:
                    assert e.evict(*arrays(addrs)) == len(removed)
                    g.insert(removed)
                else:
                    e.unset(*arrays(addrs))
            elif op == "get":
                addrs = rng.sample(pool, 20)
                if wide and len(gone) > 40:
                    old = list(dict.fromkeys(gone[:len(gone) // 2]))
                    addrs = rng.sample(old, min(len(old), 20)) + rng.sample(pool, 10)
                addrs.insert(5, addrs[1])                           # a second miss of one address finds nothing
                path = rng.choice(["batch", "dev", "small"])
                valid = None
                if path != "small" and rng.random() < 0.5:
                    valid = np.ones(len(addrs), dtype=np.uint8)
                    valid[3] = 0
                out, st = _get(E, e, path, addrs, valid)
                answers.append((out.copy(), st.copy()))
                for i, a in enumerate(addrs):
                    if valid is not None and not valid[i]:
                        assert st[i] == E.INVALID
                    elif a in store:
                        assert st[i] == E.HIT and (out[i] == store[a]).all(), (i, a, path)
                    else:
                        assert st[i] == E.MISS, (i, a, st[i], path)
                g.probe([a for i, a in enumerate(addrs) if (valid is None or valid[i]) and a not in store])
            elif op == "unset":
                addrs = rng.sample(pool, 6)
                e.unset(*arrays(addrs))
                for a in addrs:
                    store.pop(a, None)
                g.remove(addrs)
            elif op in ("inv", "inv_scan"):
                u = rng.choice((11, 12, 13))
                lo = rng.randrange(span - 10)
                hi = lo + (rng.randrange(4) if op == "inv" else 100)   # scan from 16 (1024 slots) or 64 (4096)
                e.invalidate(u, lo, hi)
                for a in [a for a in store if a[0] == u and lo <= a[1] <= hi]:
                    del store[a]
                g.remove_span(u, lo, hi)
            elif op == "rename":
                uf, ut = rng.sample((11, 12, 13), 2)
                lo = rng.randrange(span - 10)
                hi = lo + rng.randrange(10)
                moved, dropped = e.rename(uf, ut, lo, hi)
                assert dropped == 0
                for a in [a for a in store if a[0] == uf and lo <= a[1] <= hi]:
                    store[(ut, a[1])] = store.pop(a)
                g.remove_span(uf, lo, hi)
                g.remove_span(ut, lo, hi)
            elif op == "patch":
                addrs = rng.sample(pool, 4)
                st = e.patch(*arrays(addrs), [1] * 4, [b"\x5a"] * 4)
                for a, s in zip(addrs, st):
                    assert s == (E.HIT if a in store else E.MISS), (a, s)
                    if a in store:
                        store[a] = store[a].copy()
                        store[a][1] = 0x5A
            if ghost:
                _check(e, g)
        assert not ghost or (g.inserted > 20 and g.refaults > 5 and g.removed > 0), g.stats()
        assert not (ghost and wide) or (g.replaced > 0 and g.beyond > 0 and g.hist[63] + g.hist[62] > 0), g.stats()
        return answers
    finally:
        e.close()


@pytest.mark.parametrize("pshift", [12, 16, 17])
@pytest.mark.parametrize("seed", [1, 2])
def test_the_ghost_table_follows_the_model_after_every_step(E, gpu, pshift, seed):
    _sequence(E, pshift, True, seed)


@pytest.mark.parametrize("pshift", [12, 16])
@pytest.mark.parametrize("seed", [3, 4])
def test_full_sets_and_old_ghosts_follow_the_model(E, gpu, pshift, seed):
    """Sets fill and ghosts outlive the table: the oldest way is the one replaced, `replaced` counts it, and a
    refault at d >= entries goes to `beyond`, word for word as the model."""
    _sequence(E, pshift, True, seed, steps=80, wide=True)


@pytest.mark.parametrize("pshift", [12, 17])
def test_without_the_flag_the_sequence_answers_the_same(E, gpu, pshift):
    with_flag = _sequence(E, pshift, True, 7)
    without = _sequence(E, pshift, False, 7)
    assert len(with_flag) == len(without)
    for (o1, s1), (o2, s2) in zip(with_flag, without):
        assert (s1 == s2).all()
        hit = s1 == E.HIT
        assert (o1[hit] == o2[hit]).all()


def test_the_calls_need_the_flag(E, gpu):
    e = E.Engine(pshift=12, capacity=CAP, arena_bytes=64 << 20, max_batch=64)
    try:
        for call in (lambda: e.evict([1], [2]), e.ghost_stats, e.ghost_read):
            with pytest.raises(RuntimeError, match="CMB200_GHOST"):
                call()
    finally:
        e.close()


def test_the_multi_gpu_calls_are_refused(E, gpu):
    e = E.Engine(pshift=12, capacity=CAP, arena_bytes=64 << 20, max_batch=64, flags=E.GHOST)
    try:
        page = np.zeros((1, 4096), dtype=np.uint8)
        with pytest.raises(RuntimeError, match="CMB200_GHOST"):
            e.put_step([1], [2], page)
        with pytest.raises(RuntimeError, match="CMB200_GHOST"):
            e.import_records_dev(0, None, 0)
        with pytest.raises(RuntimeError, match="CMB200_GHOST"):
            e.open_peer(1, bytes(64), 1 << 20)
        assert e.ghost_stats()["inserted"] == 0
    finally:
        e.close()


def test_host_tier_laps_stamp_what_they_retire_in_tier_order(E, gpu):
    """Records of equal size demoted one by one: each lap of the ring retires the oldest, and the ghosts'
    stamps follow the demotion order."""
    bs = 1 << 12
    e = E.Engine(pshift=12, capacity=CAP, arena_bytes=64 << 20, max_batch=64, flags=E.GHOST,
                 host_tier_bytes=32 << 10)
    try:
        addrs = [(21, l) for l in range(24)]
        page = np.random.default_rng(3).integers(0, 256, size=(1, bs), dtype=np.uint8)   # stored raw: 7 per lap
        for a in addrs:
            u, l = np.array([a[0]], dtype=np.uint64), np.array([a[1]], dtype=np.uint64)
            e.put(u, l, page)
            assert e.demote(u, l) == 1
        retired = e.host_tier_stats()["retired_records"]
        st = e.ghost_stats()
        assert retired > 0 and st["inserted"] == retired == st["clock"], (retired, st)
        tab = e.ghost_read()
        live = tab[tab[:, 2] != 0]
        order = [(int(r[0]), int(r[1])) for r in live[np.argsort(live[:, 2])]]
        assert order == addrs[:retired], order[:8]
        assert sorted(int(s) for s in live[:, 2]) == list(range(1, retired + 1))
        _, status = e.get(np.array([a[0] for a in addrs], dtype=np.uint64),
                          np.array([a[1] for a in addrs], dtype=np.uint64))
        assert (status[:retired] == E.MISS).all() and (status[retired:] == E.HIT).all()
        st = e.ghost_stats()
        assert st["refaults"] == retired and st["probes"] == retired
    finally:
        e.close()


# ---- through the drop-in: the curve against a run at twice the capacity ----

DROP_CAP, KEYS, STEPS, WARMUP = 2048, 20000, 24000, 8000


def _zipf_dropin(E, d, capacity, seed):
    """ghost_model's zipf workload through cachemap_get / cachemap_put at 4 KiB pages, synchronous puts.
    -> (hit ratio after warmup, the map's cachemap_hit_curve at extra = capacity, misses looked up, the same
    two at warmup)."""
    E.binding._libc().srand(seed)
    cm = E.Cachemap(str(d), capacity, 12, 12)
    assert cm.ok
    page = np.zeros(1 << 12, dtype=np.uint8)
    hits = reads = 0
    at_warmup = None
    try:
        for t, (a, _read) in enumerate(G._reads("zipf", STEPS, seed, 0, KEYS, 0.9)):
            if t == WARMUP:
                at_warmup = cm.hit_curve([capacity])
            hit = cm.get(a[1] << 12, a[0], 0) is not None
            if not hit:
                page[:8] = np.frombuffer(np.uint64(a[1]).tobytes(), dtype=np.uint8)
                cm.put(a[1] << 12, a[0], 0, page)
            if t >= WARMUP:
                reads += 1
                hits += hit
        return hits / reads, cm.hit_curve([capacity]), at_warmup
    finally:
        cm.free()


@pytest.mark.parametrize("devices", [None, "0,0"])
def test_the_curve_at_twice_the_capacity_matches_a_run_there(E, gpu, tmp_path, monkeypatch, devices):
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_VERIFY",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_ADMIT", "CMB200_EVICT"):
        monkeypatch.delenv(k, raising=False)
    if devices:
        monkeypatch.setenv("CMB200_DEVICES", devices)
    monkeypatch.setenv("CMB200_PERSIST", "0")
    monkeypatch.setenv("CMB200_WB_SLOTS", "0")
    monkeypatch.setenv("CMB200_GHOST", "1")
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    base, (hit, misses), (hit0, misses0) = _zipf_dropin(E, tmp_path / "a", DROP_CAP, 5)
    assert misses > misses0 > 0 and hit[0] > hit0[0]
    reads = STEPS - WARMUP
    predicted = base + (int(hit[0]) - int(hit0[0])) / reads
    monkeypatch.delenv("CMB200_GHOST")
    real = _plain_run(E, tmp_path / "b", 2 * DROP_CAP, 5)
    print(f"zipf 0.9 via the drop-in: {base:.3f} at C, predicted {predicted:.3f} at 2C, real {real:.3f}")
    assert abs(predicted - real) <= ZIPF_TOL, (base, predicted, real)


ZIPF_TOL = 0.04        # the model's error on zipf (DESIGN.md §2, *Ghost entries*) plus the draws' spread


def _plain_run(E, d, capacity, seed):
    E.binding._libc().srand(seed)
    cm = E.Cachemap(str(d), capacity, 12, 12)
    assert cm.ok
    page = np.zeros(1 << 12, dtype=np.uint8)
    hits = reads = 0
    try:
        for t, (a, _read) in enumerate(G._reads("zipf", STEPS, seed, 0, KEYS, 0.9)):
            hit = cm.get(a[1] << 12, a[0], 0) is not None
            if not hit:
                page[:8] = np.frombuffer(np.uint64(a[1]).tobytes(), dtype=np.uint8)
                cm.put(a[1] << 12, a[0], 0, page)
            if t >= WARMUP:
                reads += 1
                hits += hit
        with pytest.raises(RuntimeError):
            cm.hit_curve([capacity])                        # without the flag: -1
        return hits / reads
    finally:
        cm.free()
