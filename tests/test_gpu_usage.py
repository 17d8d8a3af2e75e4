"""GPU tests of cmb200_residency / cmb200_usage_set (k_residency_keys, k_residency_scan, k_usage_list and the
grouping) and of cachemap_residency / cachemap_usage through the drop-in, against tests/usage_model.py: after
every step of the store machine, on an engine with every flag, with pins, at every page size, over two
engines, across a restart, at 2^20 records, and refused after a multi-GPU call."""
import numpy as np
import pytest

import store_machine as SM
import usage_model as UM
from test_gpu_store_machine import COARSE_SLACK_NS, Machine

pytestmark = pytest.mark.gpu

G44 = 1 << 44
FLAGS_ENV = ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_VERIFY",
             "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_ADMIT", "CMB200_EVICT", "CMB200_GHOST",
             "CMB200_ARENA_MB", "CMB200_PIN_MAX", "CMB200_KEY_FILE", "CMB200_LOAD", "CMB200_PERSIST",
             "CMB200_WB_SLOTS")


def _env(monkeypatch, **kv):
    for k in FLAGS_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in kv.items():
        monkeypatch.setenv(k, str(v))


def _strip_ts(rows):
    return [r[:9] for r in rows]


def _check_ts(got, want_lo, want_hi, slack=0):
    """oldest / newest ts of each row lie between the lowest and highest bounds the model allows."""
    for g, lo, hi in zip(got, want_lo, want_hi):
        assert lo[9] - slack <= g[9] <= hi[9] + slack, f"oldest_ts of {g[:2]}: {g[9]} not in [{lo[9]}, {hi[9]}]"
        assert lo[10] - slack <= g[10] <= hi[10] + slack, f"newest_ts of {g[:2]}: {g[10]} not in [{lo[10]}, {hi[10]}]"


# ---- 1. after every step of the store machine --------------------------------------------------------------

class UsageMachine(Machine):
    def check(self, kind):
        super().check(kind)
        m, cfg = self.m, self.cfg
        bs = cfg.bsize
        lo = {r.addr: (UM.record_len(r.clen, bs), r.host_pos is not None, r.ts_lo) for r in m.rec.values()}
        hi = {a: (n, t, m.rec[m.key(a)].ts_hi) for a, (n, t, _) in lo.items()}
        keyed = (cfg.table_slots + 2) // 64                 # cmb200_invalidate's threshold
        ranges = []
        for u in cfg.us:
            ranges.append((u, 2, 2 + keyed - 1))             # keyed: l_last - l_first < threshold
            ranges.append((u, 0, cfg.nl + keyed))            # by scan
        ranges.append((SM.PURGE_U, 0, cfg.table_slots // 8 + 24))
        for u, l in SM.edge_addrs():
            ranges.append((u, l, l))
            ranges.append((u, l - keyed, l) if l >= keyed else (u, l, l + keyed))
        for u, lf, ll in ranges:
            got = self.eng.residency(u, lf, ll)
            want = UM.engine_residency(lo, u, lf, ll)
            assert (got == want).all(), f"residency of {u} [{lf}, {ll}]: {np.flatnonzero(got != want)[:8]} differ"
        n, rows = self.E.usage_set([self.eng.h], 1 << 16)
        got = UM.as_tuples(rows)
        wn, wlo = UM.usage(lo, [], 1 << 16)
        _, whi = UM.usage(hi, [], 1 << 16)
        assert n == wn, f"usage: {n} objects, model {wn}"
        assert _strip_ts(got) == _strip_ts(wlo), "usage rows differ from the model"
        slack = COARSE_SLACK_NS if cfg.flags & SM.TOUCH else 0
        _check_ts(got, wlo, whi, slack)


@pytest.fixture
def machine_env(monkeypatch):
    def setup(cfg):
        for k in ("CMB200_SEG_KB", "CMB200_CKPT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in cfg.env:
            monkeypatch.setenv(k, v)
    return setup


@pytest.mark.parametrize("name,seed", [(n, s) for n in sorted(SM.CONFIGS) for s in SM.CONFIGS[n].seeds])
def test_usage_after_every_store_machine_step(E, gpu, oracle, tmp_path, machine_env, name, seed):
    cfg = SM.CONFIGS[name]
    machine_env(cfg)
    UsageMachine(E, oracle, cfg, seed, tmp_path).run()


# ---- 2. the calls change nothing -----------------------------------------------------------------------------

def _records(e, u, l, cap):
    """Every record's address and ts (the sampler's answer from every slot) and its stored bytes."""
    addr, ts, ok = e.sample(np.arange(cap + 2, dtype=np.uint64))
    return addr.tobytes(), ts.tobytes(), ok.tobytes(), [None if r is None else bytes(r) for r in e.read_records(u, l)]


def test_the_calls_change_nothing(E, gpu):
    n, cap = 2048, 8192
    e = E.Engine(pshift=12, capacity=cap, arena_bytes=64 << 20, table_slots=cap, max_batch=512,
                 flags=E.TOUCH | E.FREQ | E.GHOST | E.VERIFY, host_tier_bytes=8 << 20)
    try:
        rng = np.random.default_rng(3)
        u = np.repeat(np.array([5, 6, 7, 8], dtype=np.uint64), n // 4)
        l = np.tile(np.arange(n // 4, dtype=np.uint64), 4)
        e.put(u, l, rng.integers(0, 4, size=(n, 4096), dtype=np.uint8))
        e.get_small(u[:300], l[:300])
        e.get(u[::3], l[::3])
        assert e.demote(u[1000:1400], l[1000:1400]) > 0
        assert e.evict(u[1800:1900], l[1800:1900]) > 0
        e.get(u[1800:1850], l[1800:1850])                   # ghost refaults
        recs = _records(e, u, l, cap)
        # the statistics are read last before the calls and first after them
        before = (e.freq_read().tobytes(), e.ghost_read().tobytes(), sorted(e.host_tier_stats().items()),
                  sorted(e.stats().items()))
        r1 = e.residency(6, 0, n // 4 - 1)                   # scan
        r2 = e.residency(5, 0, 7)                            # keyed
        rows = e.usage()
        st = sorted(e.stats().items())
        after = (e.freq_read().tobytes(), e.ghost_read().tobytes(), sorted(e.host_tier_stats().items()), st)
        assert after == before
        assert _records(e, u, l, cap) == recs
        assert (r1 == 2).sum() > 0 and (r2 > 0).all() and len(rows) == 4
        assert int(rows["tier_pages"].sum()) == int(e.host_tier_stats()["records"])
    finally:
        e.close()


# ---- 3. pins --------------------------------------------------------------------------------------------------

def test_pinned_pages_on_keyed_and_scan_size_pin_lists(E, gpu):
    cap = 4096
    e = E.Engine(pshift=12, capacity=cap, arena_bytes=64 << 20, table_slots=cap, max_batch=512)
    try:
        n = 600
        u = np.repeat(np.array([5, 6], dtype=np.uint64), n // 2)
        l = np.concatenate([np.arange(n // 2, dtype=np.uint64), np.arange(n // 2, dtype=np.uint64) | np.uint64(G44)])
        lens = e.put(u, l, np.zeros((n, 4096), dtype=np.uint8))
        recs = {(int(a), int(b)): (UM.record_len(int(c), 4096), False, 0) for a, b, c in zip(u, l, lens)}
        for pins in ([(5, 3, 9)],                                          # 7 pages: keyed count
                     [(5, 0, 199), (6, G44 + 10, G44 + 400)]):             # past (cap + 2) / 64: scan count
            e.pin_set(pins)
            _, want = UM.usage(recs, pins, 10)
            got = UM.as_tuples(e.usage())
            assert _strip_ts(got) == _strip_ts(want)
            assert sum(r[5] for r in got) == sum(e.pin_count())
    finally:
        e.close()


def test_the_pinned_bit_through_the_drop_in(E, gpu, tmp_path, monkeypatch):
    _env(monkeypatch, CMB200_PERSIST=0, CMB200_WB_SLOTS=64)
    cm = E.Cachemap(str(tmp_path), 4096, 12, 12)
    try:
        bs = 4096
        for p in range(10):
            cm.put(p * bs, 5, 0, np.full(bs, p, dtype=np.uint8))
        assert cm.pin(5, 0, 8 * bs, 6 * bs) == 6                          # pages 8..13, 10..13 not cached
        n, vec = cm.residency(5, 0, 100, 16 * bs - 200)                     # pages 0..15, partial ends
        assert n == 10 and len(vec) == 16
        want = [E.IN_HBM] * 8 + [E.IN_HBM | E.PINNED] * 2 + [E.PINNED] * 4 + [0] * 2
        assert vec.tolist() == want
        cnt, rows = cm.usage(10)
        assert cnt == 1 and int(rows[0]["pinned_pages"]) == 2 and int(rows[0]["pages"]) == 10
        # refusals leave the vector alone
        assert cm.residency(5, 0, 0, 0)[0] == -1
        assert cm.residency(5, 0, 0, (1 << 64) - 1)[0] == -1
        assert cm.residency(5, 0, G44 << 12, 1)[0] == -1
        assert cm.residency(5, 0, (G44 - 1) << 12, 2 * bs)[0] == -1
    finally:
        cm.free()


# ---- 4. page sizes, raw records -------------------------------------------------------------------------------

@pytest.mark.parametrize("pshift", [12, 16, 17, 20])
def test_raw_records_at_every_page_size(E, gpu, pshift):
    bs = 1 << pshift
    n = 24
    e = E.Engine(pshift=pshift, accel=0, capacity=1024, arena_bytes=max(64 << 20, 4 * n * bs), max_batch=32)
    try:
        u = np.array([3] * 10 + [4] * 14, dtype=np.uint64)
        l = np.array(list(range(10)) + [G44 * 2 + k for k in range(14)], dtype=np.uint64)
        e.put(u, l, np.random.default_rng(pshift).integers(0, 256, size=(n, bs), dtype=np.uint8))
        got = UM.as_tuples(e.usage())
        assert _strip_ts(got) == [(4, 2, 0, 14, 0, 0, 14 * (24 + bs), 0, 13), (3, 0, 0, 10, 0, 0, 10 * (24 + bs), 0, 9)]
        assert e.residency(4, 2 * G44, 2 * G44 + 20).tolist() == [1] * 14 + [0] * 7
    finally:
        e.close()


# ---- 5. two engines, and a restart ----------------------------------------------------------------------------

def _fill(cm, bs, seed, values=3):
    rng = np.random.default_rng(seed)
    offs, nhs, gens = [], [], []
    for obj in range(40):
        pages = int(rng.integers(1, 40))
        offs += [p * bs for p in range(pages)]
        nhs += [1000 + obj % 13] * pages
        gens += [obj // 13] * pages
    k = len(offs)
    pages = rng.integers(0, values, size=(k, bs), dtype=np.uint8)
    # batches of 32 pages: a batch larger than a small arena would drop what the first fill leaves no room for
    for at in range(0, k, 32):
        cm.put_batch(np.array(offs[at:at + 32], dtype=np.uint64), np.array(nhs[at:at + 32], dtype=np.uint64),
                     np.array(gens[at:at + 32], dtype=np.uint32), pages[at:at + 32])
    return k


def _usage(cm):
    n, rows = cm.usage(1 << 12)
    assert n >= 0
    return UM.as_tuples(rows)


def test_one_and_two_engines_answer_alike(E, gpu, tmp_path, monkeypatch):
    got = {}
    for devices in (None, "0,0"):
        kv = {"CMB200_PERSIST": 0}
        if devices:
            kv["CMB200_DEVICES"] = devices
        _env(monkeypatch, **kv)
        d = tmp_path / (devices or "one")
        d.mkdir()
        cm = E.Cachemap(str(d), 1 << 14, 12, 12)
        try:
            k = _fill(cm, 4096, 5)
            assert len(cm.engine_handles()) == (2 if devices else 1)
            got[devices] = _usage(cm)
            assert sum(r[3] for r in got[devices]) == k
            n, vec = cm.residency(1000, 0, 0, 64 * 4096)
            assert n == int((vec & 3 != 0).sum()) > 0
            got[(devices, "res")] = vec.tolist()
        finally:
            cm.free()
    # every field but the put times, which the two maps took at different moments
    assert [r[:9] for r in got[None]] == [r[:9] for r in got["0,0"]]
    assert got[(None, "res")] == got[("0,0", "res")]


@pytest.mark.parametrize("sealed,tier", [(False, False), (True, False), (False, True)])
def test_the_answer_survives_a_restart(E, gpu, tmp_path, monkeypatch, sealed, tier):
    kv = {}
    if sealed:
        key = tmp_path / "key"
        key.write_bytes(bytes(range(32)))
        kv["CMB200_KEY_FILE"] = str(key)
    if tier:
        kv["CMB200_HOST_TIER_MB"] = 64
        kv["CMB200_ARENA_MB"] = 1
    d = tmp_path / "c"
    d.mkdir()
    _env(monkeypatch, **kv)
    cm = E.Cachemap(str(d), 1 << 14, 12, 12)
    try:
        k = _fill(cm, 4096, 9, 256 if tier else 3)            # raw 4 KiB records overflow a 1 MiB arena
        before = _usage(cm)
        assert sum(r[3] for r in before) == k
        assert cm.checkpoint() == 0
    finally:
        cm.free()
    if tier:
        # a load never evicts or demotes: an arena that holds every record keeps every page, and only where
        # they are may change
        monkeypatch.setenv("CMB200_ARENA_MB", "64")
    cm = E.Cachemap(str(d), 1 << 14, 12, 12)
    try:
        after = _usage(cm)                                   # the first call starts the map and loads the file
    finally:
        cm.free()
    if tier:
        assert sum(r[4] for r in before) > 0
        drop = lambda rs: sorted(r[:4] + r[5:] for r in rs)
        assert drop(after) == drop(before)
    else:
        assert after == before


# ---- 6. scale and determinism ----------------------------------------------------------------------------------

def test_a_million_records_in_65536_objects(E, gpu):
    n, objs = 1 << 20, 1 << 16
    rng = np.random.default_rng(17)
    # uneven sizes: a few large objects, many small ones, summing to n
    w = rng.pareto(1.2, objs) + 0.05
    sizes = np.maximum(1, np.floor(w / w.sum() * n)).astype(np.int64)
    sizes[np.argmax(sizes)] += n - sizes.sum()
    assert sizes.sum() == n and sizes.min() >= 1
    obj = np.repeat(np.arange(objs, dtype=np.uint64), sizes)
    page = np.concatenate([np.arange(s, dtype=np.uint64) for s in sizes])
    u = np.uint64(77) + obj // np.uint64(4)
    genid = obj % np.uint64(4)
    l = (genid << np.uint64(44)) | page
    ts = rng.integers(1, 1 << 60, size=n, dtype=np.uint64)
    e = E.Engine(pshift=12, capacity=n, arena_bytes=2 << 30, table_slots=1 << 21, max_batch=1 << 16)
    try:
        lens = np.zeros(n, dtype=np.int64)
        step = 1 << 16
        pages = np.zeros((step, 4096), dtype=np.uint8)
        for at in range(0, n, step):
            pages[:, :8] = np.arange(at, at + step, dtype=np.uint64).view(np.uint8).reshape(step, 8)
            lens[at:at + step] = e.put(u[at:at + step], l[at:at + step], pages, ts=ts[at:at + step])
        assert e.stats()["entries"] == n and (lens > 0).all() and (lens < 4096).all()
        stored = 24 + lens
        # numpy group-by of what was put
        key = obj
        order = np.argsort(key, kind="stable")
        starts = np.flatnonzero(np.r_[True, key[order][1:] != key[order][:-1]])
        sums = lambda a: np.add.reduceat(a[order], starts)
        want = np.zeros(objs, dtype=E.USAGE_DTYPE)
        want["nhid"] = u[order][starts]; want["genid"] = genid[order][starts]
        want["pages"] = sizes; want["stored_bytes"] = sums(stored)
        want["first_page"] = 0; want["last_page"] = sizes - 1
        want["oldest_ts"] = np.minimum.reduceat(ts[order], starts)
        want["newest_ts"] = np.maximum.reduceat(ts[order], starts)
        idx = np.lexsort((want["genid"], want["nhid"], -want["stored_bytes"].astype(np.int64)))
        want = want[idx]
        cnt, rows = E.usage_set([e.h], objs)
        assert cnt == objs
        assert rows.tobytes() == want.tobytes()
        cnt2, rows2 = E.usage_set([e.h], objs)
        assert cnt2 == cnt and rows2.tobytes() == rows.tobytes()
        cnt3, top = E.usage_set([e.h], 100)
        assert cnt3 == objs and top.tobytes() == want[:100].tobytes()
        assert E.usage_set([e.h], 0)[0] == objs
        # the largest object, keyed and by scan
        big = int(np.argmax(sizes))
        ub, gb = 77 + big // 4, big % 4
        span = max(int(sizes[big]) + 100, (1 << 21) // 64 + 1)             # past the keyed threshold: a scan
        want_res = np.zeros(span, dtype=np.uint8)
        want_res[:sizes[big]] = 1
        assert (e.residency(ub, gb << 44, (gb << 44) + span - 1) == want_res).all()
        assert e.residency(ub, gb << 44, (gb << 44) + 9).tolist() == [1] * min(10, int(sizes[big])) + [0] * max(0, 10 - int(sizes[big]))
    finally:
        e.close()


# ---- 7. refusal -------------------------------------------------------------------------------------------------

def test_refused_after_a_multi_gpu_call(E, gpu):
    e = E.Engine(pshift=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    try:
        e.put(np.full(4, 5, dtype=np.uint64), np.arange(4, dtype=np.uint64), np.zeros((4, 4096), dtype=np.uint8))
        assert e.residency(5, 0, 3).tolist() == [1, 1, 1, 1]
        e.set_stream_order(1 << 20, 2)
        with pytest.raises(RuntimeError, match="multi-GPU"):
            e.residency(5, 0, 3)
        with pytest.raises(RuntimeError, match="multi-GPU"):
            E.usage_set([e.h], 10)
    finally:
        e.close()
