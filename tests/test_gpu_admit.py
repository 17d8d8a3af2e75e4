"""GPU tests of the frequency sketch (CMB200_FREQ) and of admission by frequency (CMB200_ADMIT=freq).

Every get path counts every request with a valid address in the sketch, and the sketch read back
(cmb200_freq_read) equals tests/admit_model.py's Sketch word for word, halvings included; estimates equal the
model's; gets return the same bytes and statuses with the flag as without.  Then admission through the
drop-in on the scan workload, against the model's prediction."""
import random

import numpy as np
import pytest

import admit_model as A
import datagen
import key_edges
from oracle import snapshot

pytestmark = pytest.mark.gpu


def _engine(E, pshift, freq, capacity=64, flags=0):
    return E.Engine(pshift=pshift, capacity=capacity, arena_bytes=64 << 20, max_batch=256,
                    flags=flags | (E.FREQ if freq else 0))


def _get(E, e, path, u, l, valid=None):
    """(pages, status) of one call of a get path: the fused single-page get, the batch get to host or device."""
    u = np.asarray(u, dtype=np.uint64)
    l = np.asarray(l, dtype=np.uint64)
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


def _count(sk, u, l, valid=None):
    """The model of one counting launch."""
    sk.launch([A.fnv_addr(int(a), int(b)) for i, (a, b) in enumerate(zip(u, l)) if valid is None or valid[i]])


def _check(e, sk, u_all, l_all):
    assert (e.freq_read() == sk.words()).all()
    st = e.freq_stats()
    assert (st["width"], st["period"], st["increments"], st["since_halving"], st["halvings"]) == \
        (sk.width, sk.period, sk.increments, sk.since, sk.halvings), (st, vars(sk))
    est = e.freq_estimate(u_all, l_all)
    assert list(est) == [sk.estimate(A.fnv_addr(int(a), int(b))) for a, b in zip(u_all, l_all)]


def _store(e, pshift, count=32, u=11):
    uu = np.full(count, u, dtype=np.uint64)
    ll = np.arange(count, dtype=np.uint64)
    pages = np.stack([datagen.make_page("RTZM"[i % 4], 1 << pshift, 1 + i) for i in range(count)])
    e.put(uu, ll, pages)
    return uu, ll, pages


PATHS = [(12, ("small",)), (16, ("small",)), (17, ("small",)), (12, ("batch",)), (16, ("batch_dev",)),
         (16, ("small", "batch", "batch_dev"))]


@pytest.mark.parametrize("pshift,paths", PATHS, ids=lambda p: p if isinstance(p, int) else "+".join(p))
def test_the_sketch_counts_every_get_as_the_model_does(E, gpu, pshift, paths):
    """A seeded sequence of single requests and mixed launches (hits, misses, invalid addresses on the batch
    paths) long enough for two halvings (capacity 64: width 64, period 640).  With the flag the gets answer
    what they answer without it."""
    on, off = _engine(E, pshift, True), _engine(E, pshift, False)
    sk = A.Sketch(64)
    rng = random.Random(pshift * 7 + len(paths))
    try:
        u, l, pages = _store(on, pshift)
        _store(off, pshift)
        u_all = np.concatenate([u, np.full(16, 11, dtype=np.uint64)])
        l_all = np.concatenate([l, np.arange(1000, 1016, dtype=np.uint64)])      # 16 addresses never stored
        calls = 0
        while sk.halvings < 2:
            path = rng.choice(paths)
            n = 1 if rng.random() < 0.4 else rng.randint(2, 24)
            pick = [rng.randrange(len(u_all)) for _ in range(n)]
            cu, cl = u_all[pick], l_all[pick]
            valid = None
            if path != "small" and rng.random() < 0.3:
                valid = np.array([rng.random() < 0.7 for _ in range(n)], dtype=np.uint8)
            got, st = _get(E, on, path, cu, cl, valid)
            ref, st_off = _get(E, off, path, cu, cl, valid)
            assert (st == st_off).all(), (st, st_off)
            assert (got[st == E.HIT] == ref[st_off == E.HIT]).all()
            for i, k in enumerate(pick):
                want = E.INVALID if valid is not None and not valid[i] else (E.HIT if k < len(u) else E.MISS)
                assert st[i] == want, (i, st)
                if want == E.HIT:
                    assert (got[i] == pages[k]).all()
            _count(sk, cu, cl, valid)
            calls += 1
            if calls % 17 == 0:
                _check(on, sk, u_all, l_all)
        _check(on, sk, u_all, l_all)
    finally:
        on.close()
        off.close()


@pytest.mark.parametrize("path", ["small", "batch"])
def test_bad_entries_and_sentinel_keys_count(E, gpu, path):
    fx = key_edges.load()
    g = fx["groups"]
    stored = [g["pair0"][0], g["quad"][0], g["key0"][0], g["key_ones"][0]]
    others = [g["pair0"][1], g["quad"][1], g["quad"][2], g["key0"][1], g["key_ones"][1]]
    e = _engine(E, 16, True)
    sk = A.Sketch(64)
    try:
        u = np.array([a[0] for a in stored], dtype=np.uint64)
        l = np.array([a[1] for a in stored], dtype=np.uint64)
        e.put(u, l, np.stack([datagen.make_page("T", 1 << 16, 40 + i) for i in range(len(u))]))
        ou = np.array([a[0] for a in others], dtype=np.uint64)
        ol = np.array([a[1] for a in others], dtype=np.uint64)
        for _ in range(3):
            _, st = _get(E, e, path, ou, ol)
            assert (st == E.BAD_ENTRY).all(), st
            _count(sk, ou, ol)
            _, st = _get(E, e, path, u, l)
            assert (st == E.HIT).all(), st
            _count(sk, u, l)
        _check(e, sk, np.concatenate([u, ou]), np.concatenate([l, ol]))
        assert e.freq_estimate(u[2:], l[2:]).min() >= 3          # keys 0 and ~0 are counted like any other
    finally:
        e.close()


@pytest.mark.parametrize("pshift,path", [(16, "small"), (17, "small"), (16, "batch")])
def test_corrupt_answers_count(E, gpu, tmp_path, pshift, path):
    """CMB200_VERIFY: a page whose stored fingerprint no longer matches is answered CMB200_CORRUPT, and the
    request counts as any other."""
    good, bad = str(tmp_path / "good.snap"), str(tmp_path / "bad.snap")
    e = _engine(E, pshift, False, flags=E.VERIFY)
    try:
        u, l, pages = _store(e, pshift, count=8)
        assert e.save(good) == len(u)
    finally:
        e.close()
    ps, _flags, recs = snapshot.read_snapshot(good)
    damaged = 5
    out = [(ts, hi, lo ^ 1 if int.from_bytes(rec[8:16], "little") == damaged else lo, rec) for ts, hi, lo, rec in recs]
    snapshot.write_snapshot(bad, ps, out, with_fingerprints=True)
    e = _engine(E, pshift, True, flags=E.VERIFY)
    sk = A.Sketch(64)
    try:
        assert e.load(bad) == len(u)
        for _ in range(2):
            got, st = _get(E, e, path, u, l)
            clean = np.arange(len(u)) != damaged
            assert st[damaged] == E.CORRUPT and (st[clean] == E.HIT).all(), st
            assert (got[clean] == pages[clean]).all()
            _count(sk, u, l)
        _check(e, sk, u, l)
    finally:
        e.close()


def test_halving_happens_at_exactly_the_period(E, gpu):
    e = _engine(E, 16, True, capacity=16)          # width 16, period 160
    sk = A.Sketch(16)
    try:
        u, l, _ = _store(e, 16, count=8)
        for t in range(159):
            _get(E, e, "small", u[t % 8:t % 8 + 1], l[t % 8:t % 8 + 1])
            _count(sk, u[t % 8:t % 8 + 1], l[t % 8:t % 8 + 1])
        assert e.freq_stats()["halvings"] == 0 and e.freq_stats()["since_halving"] == 159
        _check(e, sk, u, l)
        _get(E, e, "batch", u[:1], l[:1])
        _count(sk, u[:1], l[:1])
        assert sk.halvings == 1 and e.freq_stats()["halvings"] == 1 and e.freq_stats()["since_halving"] == 0
        _check(e, sk, u, l)
    finally:
        e.close()


def test_lookups_and_reads_do_not_count(E, gpu):
    e = _engine(E, 16, True)
    try:
        u, l, _ = _store(e, 16, count=8)
        e.locate(u, l)
        e.read_records(u, l)
        e.sample(np.arange(64, dtype=np.uint64))
        e.freq_estimate(u, l)
        assert e.freq_stats()["increments"] == 0
        assert not e.freq_read().any()
    finally:
        e.close()


def test_the_multi_gpu_calls_are_refused(E, gpu):
    e = _engine(E, 16, True)
    try:
        u, l, pages = np.full(2, 5, dtype=np.uint64), np.arange(2, dtype=np.uint64), np.zeros((2, 1 << 16), np.uint8)
        rec = e.dev_alloc(2 * 32)
        try:
            with pytest.raises(RuntimeError, match="CMB200_FREQ"):
                e.put_step(u, l, pages, records_dev=rec)
            with pytest.raises(RuntimeError, match="CMB200_FREQ"):
                e.import_records_dev(2, rec, 0)
        finally:
            e.dev_free(rec)
        with pytest.raises(RuntimeError, match="CMB200_FREQ"):
            e.open_peer(1, bytes(64), 1 << 20)
        assert _get(E, e, "small", u, l)[1].tolist() == [E.MISS, E.MISS]      # the engine still serves
    finally:
        e.close()
    off = _engine(E, 16, False)
    try:
        with pytest.raises(RuntimeError, match="CMB200_FREQ"):
            off.freq_stats()
    finally:
        off.close()


# ---- admission through the drop-in ---------------------------------------------------------------

def _estimate(E, handle, u, l) -> int:
    addr = np.array([[u, l]], dtype=np.uint64)
    est = np.zeros(1, dtype=np.uint8)
    assert E.lib().cmb200_freq_estimate(handle, 1, addr.ctypes.data, est.ctypes.data) == 0, E.last_error()
    return int(est[0])


def _version(p, v):
    page = np.full(1 << 12, (p * 7 + v) % 251, dtype=np.uint8)
    page[:16] = np.frombuffer(np.array([p, v], dtype=np.uint64).tobytes(), dtype=np.uint8)
    return page


@pytest.mark.parametrize("ring", [True, False], ids=["ring", "sync"])
@pytest.mark.parametrize("how", ["put", "put_batch"])
def test_a_rejected_page_never_serves_its_old_version(E, gpu, tmp_path, monkeypatch, ring, how):
    """A map at capacity, pages 0..511 read twice, pages 512.. never: new versions of cached pages whose
    estimate is 0 lose to every victim.  After the puts (and the ring's flush) a get returns the new version
    or nothing, never the old one; a page rejected at capacity is not served at all."""
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_VERIFY",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_EVICT", "CMB200_WB_SLOTS"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("CMB200_PERSIST", "0")
    monkeypatch.setenv("CMB200_ADMIT", "freq")
    if not ring:
        monkeypatch.setenv("CMB200_WB_SLOTS", "0")
    nhid, cap = 77, 1024
    cm = E.Cachemap(str(tmp_path), cap, 12, 12)
    assert cm.ok
    try:
        for p in range(cap):
            cm.put(p << 12, nhid, 0, _version(p, 1))
        h = cm.engine_handle()                         # every put has landed
        for _ in range(2):
            for p in range(cap // 2):
                assert cm.get(p << 12, nhid, 0) == _version(p, 1).tobytes()
        h = cm.engine_handle()
        assert E.engine_stats(h)["entries"] == cap     # nothing evicted: pages 512.. are cached, never read
        cands = [p for p in range(cap // 2, cap) if _estimate(E, h, nhid, p) == 0][:4]
        assert len(cands) == 4
        new = np.stack([_version(p, 2) for p in cands])
        if how == "put":
            for p, pg in zip(cands, new):
                cm.put(p << 12, nhid, 0, pg)
        else:
            cm.put_batch(np.array([p << 12 for p in cands], dtype=np.uint64), np.full(4, nhid, dtype=np.uint64),
                         np.zeros(4, dtype=np.uint32), new)
        cm.engine_handles()                            # the ring has flushed
        got = [cm.get(p << 12, nhid, 0) for p in cands]
        for p, g in zip(cands, got):
            assert g != _version(p, 1).tobytes(), p
            assert g is None or g == _version(p, 2).tobytes(), p
        assert got[0] is None
        admitted, rejected = cm.admission()
        assert rejected >= 1 and admitted == 0, (admitted, rejected)
        if how == "put_batch":
            assert all(g is None for g in got) and rejected == 4
    finally:
        cm.free()
# Synchronous puts (no write-behind ring), so that every get reaches the GPU and is counted, as the model
# counts it, and every put at capacity is one admission decision (TinyLFU over the store's sampler).

CAPACITY, HOT, STEPS, WARMUP = 4096, 2048, 16384, 8192
SEEDS = (1, 2, 3)


def _scan_dropin(E, d, seed):
    """admit_model.scan through cachemap_get / cachemap_put at 4 KiB pages, one scan page per hot read."""
    E.binding._libc().srand(seed)
    cm = E.Cachemap(str(d), CAPACITY, 12, 12)
    assert cm.ok
    rng = random.Random(seed ^ 0x5CA7)
    page = np.zeros(1 << 12, dtype=np.uint8)
    hits = reads = nxt = 0
    try:
        for t in range(STEPS):
            h = rng.randrange(HOT)
            hit = cm.get(h << 12, A.HOT_NHID, 0) is not None
            if not hit:
                page[:8] = np.frombuffer(np.uint64(h).tobytes(), dtype=np.uint8)
                cm.put(h << 12, A.HOT_NHID, 0, page)
            if cm.get(nxt << 12, A.COLD_NHID, 0) is None:
                page[:8] = np.frombuffer(np.uint64(nxt).tobytes(), dtype=np.uint8)
                cm.put(nxt << 12, A.COLD_NHID, 0, page)
            nxt += 1
            if t >= WARMUP:
                reads += 1
                hits += hit
        adm = cm.admission()
    finally:
        cm.free()
    return hits / reads, adm


@pytest.mark.parametrize("devices", [None, "0,0"])
def test_admission_keeps_the_hot_set_through_a_scan_as_the_model_says(E, gpu, tmp_path, monkeypatch, devices):
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_VERIFY",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        monkeypatch.delenv(k, raising=False)
    if devices:
        monkeypatch.setenv("CMB200_DEVICES", devices)
    g = 2 if devices else 1
    monkeypatch.setenv("CMB200_PERSIST", "0")
    monkeypatch.setenv("CMB200_WB_SLOTS", "0")
    monkeypatch.setenv("CMB200_EVICT", "access")
    got, model = {}, {}
    for admit in ("all", "freq"):
        monkeypatch.setenv("CMB200_ADMIT", admit)
        runs = []
        for seed in SEEDS:
            d = tmp_path / f"{admit}{seed}"
            d.mkdir()
            runs.append(_scan_dropin(E, d, seed))
        got[admit] = float(np.mean([r for r, _ in runs]))
        adm = [a for _, a in runs]
        if admit == "all":
            assert all(a == (0, 0) for a in adm), adm
        else:
            assert all(a[0] > 0 and a[1] > 0 for a in adm), adm
        model[admit] = float(np.mean([A.scan(True, admit == "freq", CAPACITY, HOT, 1, STEPS, WARMUP, seed=s, table=True,
                                             engines=g) for s in SEEDS]))
    print("scan hot-set hit ratio, drop-in vs TableStore model:", got, model)
    assert abs(got["freq"] - model["freq"]) <= 0.01, (got, model)
    assert abs(got["all"] - model["all"]) <= 0.03, (got, model)
    assert got["freq"] > got["all"] + 0.2, got
