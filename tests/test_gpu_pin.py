"""GPU tests of pinned pages: cmb200_pin_set's filter in the sampler (k_sample_pin, k_sample_scan_pin), the
pinned records' counts and promotion (k_pin_select on its keyed and its scan path), and cachemap_pin through
the drop-in: a flood of puts under every eviction, admission, ghost, host-tier and device setting leaves every
pinned page cached, and the pins survive a restart, move with a rename and outlive an invalidation."""
import ctypes as C
import os
import time

import numpy as np
import pytest

import key_edges as K
import pin_model as PM

pytestmark = pytest.mark.gpu

TO_END = (1 << 64) - 1
FLAGS_ENV = ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_VERIFY",
             "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_ADMIT", "CMB200_EVICT", "CMB200_GHOST",
             "CMB200_ARENA_MB", "CMB200_PIN_MAX", "CMB200_KEY_FILE", "CMB200_LOAD", "CMB200_PERSIST",
             "CMB200_WB_SLOTS")


def _pages(n, bsize, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n, bsize), dtype=np.uint8)


def _filled_engine(E, n, u=7, pshift=12, **kw):
    e = E.Engine(pshift=pshift, capacity=kw.pop("capacity", 4096), arena_bytes=kw.pop("arena_bytes", 64 << 20),
                 max_batch=512, **kw)
    lv = np.arange(n, dtype=np.uint64)
    e.put(np.full(n, u, dtype=np.uint64), lv, np.zeros((n, 1 << pshift), dtype=np.uint8))
    return e


def _answers(e, r):
    addr, ts, ok = e.sample(r)
    return [(int(a[0]), int(a[1])) if k > 0 else None for a, k in zip(addr, ok)]


@pytest.mark.parametrize("frac", [0.0, 1 / 8, 1 / 2, 0.9])
def test_the_pinned_sampler_answers_the_unpinned_one_where_that_one_is_not_pinned(E, gpu, frac):
    n = 3000
    e = _filled_engine(E, n)
    try:
        rng = np.random.default_rng(int(frac * 1000) + 1)
        r = rng.integers(0, 1 << 63, size=3 * 4096, dtype=np.uint64) * 2 + 1
        base = _answers(e, r)
        assert all(a is not None for a in base)
        pinned = {int(x) for x in rng.choice(n, size=int(frac * n), replace=False)}
        ranges = PM.ranges_of(7, sorted(pinned)) + [(8, 0, 1 << 40)]   # u = 8 holds nothing
        e.pin_set(ranges)
        got = _answers(e, r)
        live = {(7, l) for l in range(n)}
        for b, g in zip(base, got):
            if b[1] not in pinned:
                assert g == b
            else:
                assert g is not None and g in live and g[1] not in pinned and g != b
        e.pin_set([])
        assert _answers(e, r) == base                  # the empty list is the unfiltered sampler
    finally:
        e.close()


def test_the_scan_fallback_finds_the_one_unpinned_record_and_none_when_all_are_pinned(E, gpu):
    e = _filled_engine(E, 5, capacity=1 << 16)
    try:
        assert e.stats()["table_slots"] >= 1 << 16     # 5 records in 65536+ slots: most walks find nothing
        r = np.random.default_rng(3).integers(0, 1 << 63, size=4096, dtype=np.uint64)
        e.pin_set([(7, 0, 2), (7, 4, 4)])
        assert set(_answers(e, r)) == {(7, 3)}
        e.pin_set([(7, 0, 4)])
        assert _answers(e, r) == [None] * len(r)
    finally:
        e.close()


def test_a_pin_names_an_address_not_its_key(E, gpu):
    group = K.load()["groups"]["quad"]                 # four addresses with one store key
    e = E.Engine(pshift=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    try:
        r = np.random.default_rng(4).integers(0, 1 << 63, size=256, dtype=np.uint64)
        a, b = group[0], group[1]
        e.pin_set(PM.normalize([(b[0], b[1], b[1])]))
        e.put(np.array([a[0]], dtype=np.uint64), np.array([a[1]], dtype=np.uint64), np.zeros((1, 4096), np.uint8))
        assert set(_answers(e, r)) == {a}              # the key's record is a's: evictable
        e.put(np.array([b[0]], dtype=np.uint64), np.array([b[1]], dtype=np.uint64), np.zeros((1, 4096), np.uint8))
        assert _answers(e, r) == [None] * len(r)       # now it holds b, which is pinned
    finally:
        e.close()


@pytest.mark.parametrize("keyed", [True, False])
def test_counts_follow_the_model_on_both_paths(E, gpu, keyed):
    n = 2000
    e = _filled_engine(E, n, host_tier_bytes=64 << 20)
    try:
        cap = e.stats()["table_slots"]
        limit = (cap + 2) // 64
        tier = list(range(0, n, 7))
        assert e.demote(np.full(len(tier), 7, dtype=np.uint64), np.array(tier, dtype=np.uint64)) == len(tier)
        if keyed:
            ranges = PM.normalize([(7, 100, 100 + limit // 2 - 1), (7, 1990, 2100), (9, 0, 3)])
            assert PM.pages(ranges) <= limit
        else:
            ranges = PM.normalize([(7, 100, 100 + limit), (7, 1500, 1 << 44), (9, 0, 3)])
            assert PM.pages(ranges) > limit
        stored = {(7, l) for l in range(n)}
        pinned = {a for a in stored if PM.has(ranges, a)}
        e.pin_set(ranges)
        t = {(7, l) for l in tier}
        assert e.pin_count() == (len(pinned - t), len(pinned & t))
    finally:
        e.close()


def test_promotion_moves_pinned_tier_records_while_the_arena_has_room(E, gpu):
    bs = 4096
    e = E.Engine(pshift=12, capacity=8192, arena_bytes=4 << 20, max_batch=256, host_tier_bytes=64 << 20)
    try:
        u = np.full(400, 7, dtype=np.uint64)
        lv = np.arange(400, dtype=np.uint64)
        e.put(u, lv, _pages(400, bs, 1))
        e.demote(u[:100], lv[:100])
        e.pin_set([(7, 0, 49)])
        assert e.pin_count() == (0, 50)
        assert e.pin_promote() == 50
        assert e.pin_count() == (50, 0)
        # the tier again, then an arena that puts fill to the end: nothing moves
        e.demote(u[:50], lv[:50])
        more = 2000
        e.put(np.full(more, 8, dtype=np.uint64), np.arange(more, dtype=np.uint64), _pages(more, bs, 2))
        assert e.stats()["dropped_puts"] > 0
        assert e.pin_promote() == 0
        assert e.pin_count() == (0, 50)
    finally:
        e.close()


def test_pin_set_refuses_unsorted_or_overlapping_ranges(E, gpu):
    e = E.Engine(pshift=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    try:
        for bad in ([(7, 5, 9), (7, 0, 3)], [(7, 0, 5), (7, 5, 9)], [(7, 9, 5)]):
            with pytest.raises(RuntimeError):
                e.pin_set(bad)
        e.pin_set([(7, 0, 5), (7, 6, 9), (8, 0, 0)])   # touching is allowed at this level
    finally:
        e.close()


# ---- the drop-in ------------------------------------------------------------------------------------

CAP, PIN = 1024, 64                 # 1024: the smallest capacity cachemap_create takes


def _env(monkeypatch, **kv):
    for k in FLAGS_ENV:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("CMB200_WB_SLOTS", "0")
    for k, v in kv.items():
        monkeypatch.setenv(k, str(v))


def _put(cm, nhid, pages_l, pages):
    n = len(pages_l)
    cm.put_batch(np.array(pages_l, dtype=np.uint64) << np.uint64(cm.pshift), np.full(n, nhid, dtype=np.uint64),
                 np.zeros(n, dtype=np.uint32), pages)


def _read(cm, nhid, pages_l):
    n = len(pages_l)
    return cm.get_batch(np.array(pages_l, dtype=np.uint64) << np.uint64(cm.pshift), np.full(n, nhid, dtype=np.uint64),
                        np.zeros(n, dtype=np.uint32))


def _flood(cm, seed, n=4 * CAP, nhid=99, batch=256):
    for at in range(0, n, batch):
        _put(cm, nhid, list(range(at, at + batch)), _pages(batch, cm.bsize, seed * 1000 + at))


def _tier_state(E, cm):
    hits, hot = 0, set()
    for h in cm.engine_handles():
        hits += E.host_tier_stats(h)["hits"]
        addr = np.zeros((4096, 2), dtype=np.uint64)
        n, lost = C.c_size_t(0), C.c_uint64(0)
        E.lib().cmb200_host_tier_hot(h, 4096, addr.ctypes.data, C.byref(n), C.byref(lost))
        hot |= {(int(a[0]), int(a[1])) for a in addr[:n.value]}
    return hits, hot


@pytest.mark.parametrize("pshift", [12, 16])
@pytest.mark.parametrize("devices", [None, "0,0"])
@pytest.mark.parametrize("tier", [False, True])
@pytest.mark.parametrize("ghost", [0, 1])
@pytest.mark.parametrize("evict", ["put", "access"])
@pytest.mark.parametrize("admit", ["all", "freq"])
def test_a_flood_never_takes_a_pinned_page(E, gpu, tmp_path, monkeypatch, pshift, devices, tier, ghost, evict, admit):
    bs = 1 << pshift
    kv = dict(CMB200_PERSIST=0, CMB200_ADMIT=admit, CMB200_EVICT=evict, CMB200_GHOST=ghost)
    if devices:
        kv["CMB200_DEVICES"] = devices
    if tier:
        # an arena of about half the capacity: the flood demotes
        kv.update(CMB200_HOST_TIER_MB=max(16, 4 * CAP * bs >> 20), CMB200_ARENA_MB=max(1, CAP * bs // 2 >> 20))
    _env(monkeypatch, **kv)
    cm = E.Cachemap(str(tmp_path), CAP, 12, pshift)
    assert cm.ok
    try:
        want = _pages(PIN, bs, 7)
        assert cm.pin(5, 0, 0, PIN * bs) == PIN
        _put(cm, 5, list(range(PIN)), want)
        out, hit = _read(cm, 5, list(range(PIN)))
        assert hit.all() and (out == want).all()
        hits0, _ = _tier_state(E, cm)
        _flood(cm, pshift + 2 * tier + ghost)
        out, hit = _read(cm, 5, list(range(PIN)))
        assert hit.all() and (out == want).all()
        assert cm.pin_stats() == (PIN, PIN, 0)
        if tier:
            hits1, hot = _tier_state(E, cm)
            assert hits1 == hits0                      # the reads above were served from HBM
            assert not any(a[0] == 5 for a in hot)
        # the flood filled the map: eviction and (with the tier) demotion ran
        assert sum(E.engine_stats(h)["entries"] for h in cm.engine_handles()) <= CAP
    finally:
        cm.free()


def test_pins_promote_what_was_demoted_before_them(E, gpu, tmp_path, monkeypatch):
    _env(monkeypatch, CMB200_PERSIST=0, CMB200_HOST_TIER_MB=64)
    cm = E.Cachemap(str(tmp_path), 4096, 12, 12)
    try:
        _put(cm, 5, list(range(100)), _pages(100, 4096, 1))
        h = cm.engine_handle()
        addr = np.array([[5, l] for l in range(100)], dtype=np.uint64)
        got = C.c_uint64()
        E.lib().cmb200_demote_batch(h, 100, addr.ctypes.data, C.byref(got))
        assert got.value == 100
        assert cm.pin_stats() == (0, 0, 0)
        assert cm.pin(5, 0, 0, 40 * 4096) == 40
        assert cm.pin_stats() == (40, 40, 0)
    finally:
        cm.free()


@pytest.mark.parametrize("sealed", [False, True])
def test_pins_survive_a_restart(E, gpu, tmp_path, monkeypatch, sealed):
    kv = {}
    if sealed:
        key = tmp_path / "key"
        key.write_bytes(bytes(range(32)))
        kv["CMB200_KEY_FILE"] = str(key)
    d = tmp_path / "c"
    d.mkdir()
    _env(monkeypatch, **kv)
    bs = 4096
    want = _pages(PIN, bs, 9)
    cm = E.Cachemap(str(d), CAP, 12, 12)
    assert cm.ok
    assert cm.pin(5, 0, 0, PIN * bs) == PIN
    _put(cm, 5, list(range(PIN)), want)
    cm.free()
    raw = (d / "cachemap_b200.pins").read_bytes()
    assert raw[:8] == (b"CMB200Q1" if sealed else b"CMB200P1")
    for background in (False, True):
        if background:
            monkeypatch.setenv("CMB200_LOAD", "background")
        cm = E.Cachemap(str(d), CAP, 12, 12)
        try:
            # the list is read before the first record loads (a background load drops what does not fit the
            # arena, pinned or not, so the flood waits for it to end)
            assert cm.pin_stats()[0] == PIN
            while cm.load_progress()[0]:
                time.sleep(0.01)
            _flood(cm, 5 + background, nhid=98)
            out, hit = _read(cm, 5, list(range(PIN)))
            assert hit.all() and (out == want).all()
            assert cm.pin_stats() == (PIN, PIN, 0)
        finally:
            cm.free()
    if sealed:
        p = d / "cachemap_b200.pins"
        b = bytearray(p.read_bytes())
        b[40] ^= 1
        p.write_bytes(bytes(b))
        monkeypatch.delenv("CMB200_LOAD")
        cm = E.Cachemap(str(d), CAP, 12, 12)
        try:
            assert cm.pin_stats()[0] == 0              # the tag fails: no pins
        finally:
            cm.free()


def test_pins_move_with_a_rename_and_outlive_an_invalidation(E, gpu, tmp_path, monkeypatch):
    _env(monkeypatch, CMB200_PERSIST=0)
    bs = 4096
    want = _pages(PIN, bs, 11)
    cm = E.Cachemap(str(tmp_path), CAP, 12, 12)
    assert cm.ok
    try:
        assert cm.pin(5, 0, 0, PIN * bs) == PIN
        assert cm.pin(6, 0, 0, 8 * bs) == 8            # `to`'s own pins go
        _put(cm, 5, list(range(PIN)), want)
        assert cm.rename(5, 6, 0) == PIN
        assert cm.pin_stats() == (PIN, PIN, 0)
        assert cm.unpin(5, 0, 0, TO_END) == 0
        _flood(cm, 1)
        out, hit = _read(cm, 6, list(range(PIN)))
        assert hit.all() and (out == want).all()
        assert cm.invalidate(6, 0, 0, TO_END) == PIN
        assert cm.pin_stats() == (PIN, 0, 0)
        _put(cm, 6, list(range(PIN)), want)
        _flood(cm, 2)
        out, hit = _read(cm, 6, list(range(PIN)))
        assert hit.all() and cm.pin_stats() == (PIN, PIN, 0)
    finally:
        cm.free()
