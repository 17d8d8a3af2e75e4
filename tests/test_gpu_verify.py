"""GPU tests of the verified read mode (CMB200_VERIFY): every page a get serves is compared on the device
with the EF128 stored for its record version; a page that differs is CMB200_CORRUPT, never a hit."""
import threading

import numpy as np
import pytest

import datagen
from oracle import snapshot

pytestmark = pytest.mark.gpu


def _engine(E, pshift, verify=True, accel=12, tier=0, capacity=2048):
    return E.Engine(pshift=pshift, accel=accel, capacity=capacity, arena_bytes=256 << 20,
                    flags=E.VERIFY if verify else 0, host_tier_bytes=tier)


def _pages(kinds, n, count, seed):
    return np.stack([datagen.make_page(kinds[i % len(kinds)], n, seed + i) for i in range(count)])


def _keys(count, base=0):
    u = np.full(count, 7, dtype=np.uint64)
    l = np.arange(base, base + count, dtype=np.uint64)
    return u, l


def _get_all(E, e, u, l, pshift):
    """status and pages of every call that serves this page size: batch to host, batch to device,
    and the fused single-page get."""
    out = {}
    pages, st = e.get(u, l)
    out["batch"] = (pages, st)
    n, bsize = len(u), 1 << pshift
    dev = E.lib().cmb200_dev_alloc(e.h, n * bsize)
    try:
        st_d = np.zeros(n, dtype=np.int32)
        addr = np.stack([u, l], axis=1).astype(np.uint64)
        assert E.lib().cmb200_get_batch_dev(e.h, n, addr.ctypes.data, None, dev, st_d.ctypes.data) == 0
        host = np.zeros((n, bsize), dtype=np.uint8)
        assert E.lib().cmb200_memcpy_d2h(e.h, host.ctypes.data, dev, n * bsize) == 0
        out["batch_dev"] = (host, st_d)
    finally:
        E.lib().cmb200_dev_free(e.h, dev)
    if pshift <= 17:
        out["small"] = e.get_small(u, l)
    return out


@pytest.mark.parametrize("pshift", list(range(6, 21)))
def test_clean_pages_verify(E, gpu, pshift):
    n = 1 << pshift
    count = 12 if pshift <= 17 else 4
    for accel in (12, 0):                                  # 0: raw records, clen 0
        e = _engine(E, pshift, accel=accel)
        try:
            pages = _pages("RTZM", n, count, 100 * pshift + accel)
            u, l = _keys(count)
            e.put(u, l, pages)
            served = 0
            for call, (got, st) in _get_all(E, e, u, l, pshift).items():
                assert (st == E.HIT).all(), (pshift, accel, call, st)
                assert (got == pages).all(), (pshift, accel, call)
                served += count
            vs = e.verify_stats()
            assert vs["verified"] == served and vs["unverified"] == 0 and vs["corrupt"] == 0, (pshift, accel, vs)
        finally:
            e.close()


def _verified_round(E, e, u, l, pages, pshift, what):
    before = e.verify_stats()
    got, st = e.get(u, l)
    assert (st == E.HIT).all() and (got == pages).all(), what
    got, st = e.get_small(u, l)
    assert (st == E.HIT).all() and (got == pages).all(), what
    vs = e.verify_stats()
    assert vs["verified"] - before["verified"] == 2 * len(u), (what, vs, before)
    assert vs["unverified"] == before["unverified"] and vs["corrupt"] == 0, (what, vs)


@pytest.mark.parametrize("pshift", [16, 17])
def test_tags_follow_the_record(E, gpu, oracle, tmp_path, pshift):
    n, count = 1 << pshift, 64
    e = _engine(E, pshift, tier=256 << 20, capacity=256)
    try:
        pages = _pages("RTZM", n, count, 7000 + pshift)
        u, l = _keys(count)
        e.put(u, l, pages)
        fps, ok = e.read_fingerprints(u, l)
        assert ok.all()
        assert [tuple(int(x) for x in f) for f in fps] == [oracle.fingerprint128(p) for p in pages]
        # garbage, then compaction moves every record
        e.put(u[:16], l[:16], pages[:16])
        assert e.compact() > 0
        _verified_round(E, e, u, l, pages, pshift, "compact")
        assert e.demote(u[::2], l[::2]) == count // 2
        _verified_round(E, e, u, l, pages, pshift, "demote")
        assert e.promote(u[::2], l[::2]) == count // 2
        _verified_round(E, e, u, l, pages, pshift, "promote")
        # deleted keys past 1/8 of the table: the next compaction rebuilds it
        slots = E.engine_stats(e.h)["table_slots"]
        du, dl = _keys(slots // 8 + 64, base=1 << 20)
        filler = np.zeros((len(du), n), dtype=np.uint8)
        e.put(du, dl, filler)
        e.unset(du, dl)
        assert E.engine_stats(e.h)["tombstones"] > slots // 8
        e.compact()
        assert E.engine_stats(e.h)["tombstones"] == 0
        _verified_round(E, e, u, l, pages, pshift, "rebuild")
        path = str(tmp_path / "s.snap")
        assert e.save(path) == count
        e2 = _engine(E, pshift)
        try:
            assert e2.load(path) == count
            _verified_round(E, e2, u, l, pages, pshift, "load")
            assert (e2.read_fingerprints(u, l)[0] == fps).all()
        finally:
            e2.close()
    finally:
        e.close()


def _first_literal(payload: bytes) -> int:
    """Index of the first literal byte of an LZ4 block (the first sequence's literals)."""
    tok = payload[0]
    lit, i = tok >> 4, 1
    if lit == 15:
        while True:
            b = payload[i]
            i += 1
            lit += b
            if b != 255:
                break
    assert lit >= 1
    return i


def _corrupt_snapshot(E, pshift, path, bad_path, with_fp=True):
    """A store of R/T pages saved to `path`; `bad_path` has one literal byte of a T record and one of
    an R record flipped and the stored fingerprint of a third record changed.  -> (u, l, pages,
    indices of the three damaged keys)"""
    n, count = 1 << pshift, 24
    e = _engine(E, pshift)
    try:
        pages = _pages("RT", n, count, 9100 + pshift)
        u, l = _keys(count)
        lens = e.put(u, l, pages)
        assert (lens > 0).all()                            # R pages too: one block of literals
        assert e.save(path) == count
    finally:
        e.close()
    ps, flags, recs = snapshot.read_snapshot(path)
    by_l = {int.from_bytes(r[3][8:16], "little"): k for k, r in enumerate(recs)}
    t_i, r_i, f_i = 3, 4, 6
    out = list(recs)
    ts, hi, lo, rec = out[by_l[t_i]]
    rec = bytearray(rec)
    rec[24 + _first_literal(bytes(rec[24:]))] ^= 0x40
    out[by_l[t_i]] = (ts, hi, lo, bytes(rec))
    ts, hi, lo, rec = out[by_l[r_i]]
    rec = bytearray(rec)
    rec[24 + _first_literal(bytes(rec[24:])) + 1000] ^= 0x01   # inside the R block's one literal run
    out[by_l[r_i]] = (ts, hi, lo, bytes(rec))
    ts, hi, lo, rec = out[by_l[f_i]]
    out[by_l[f_i]] = (ts, hi, lo ^ 1, rec)
    snapshot.write_snapshot(bad_path, ps, out, with_fingerprints=with_fp)
    return u, l, pages, [t_i, r_i, f_i]


@pytest.mark.parametrize("pshift", [16, 17])
def test_corruption_is_caught_on_every_path(E, gpu, tmp_path, pshift):
    good, bad = str(tmp_path / "good.snap"), str(tmp_path / "bad.snap")
    u, l, pages, damaged = _corrupt_snapshot(E, pshift, good, bad)
    clean = np.ones(len(u), dtype=bool)
    clean[damaged] = False
    # without the flag the damaged bytes are served as hits: the gap this mode closes
    e = _engine(E, pshift, verify=False)
    try:
        e.load(bad)
        got, st = e.get(u, l)
        assert (st == E.HIT).all()
        assert not (got[damaged[0]] == pages[damaged[0]]).all() and not (got[damaged[1]] == pages[damaged[1]]).all()
        assert e.verify_stats() == dict.fromkeys(e.verify_stats(), 0)
    finally:
        e.close()
    e = _engine(E, pshift, tier=256 << 20)
    try:
        assert e.load(bad) == len(u)
        for where in ("hbm", "tier"):
            if where == "tier":
                assert e.demote(u, l) == len(u)
            got, st = e.get(u, l)
            assert (st[damaged] == E.CORRUPT).all(), (where, st)
            assert (st[clean] == E.HIT).all() and (got[clean] == pages[clean]).all(), where
            got, st = e.get_small(u, l)
            assert (st[damaged] == E.CORRUPT).all(), (where, st)
            assert (st[clean] == E.HIT).all() and (got[clean] == pages[clean]).all(), where
        vs = e.verify_stats()
        assert vs["corrupt"] == 4 * len(damaged) and vs["unverified"] == 0, vs
        bu, bl, n_bad, checked = e.verify_store()
        assert n_bad == len(damaged) and checked == len(u)
        assert sorted(int(x) for x in bl) == sorted(int(l[k]) for k in damaged) and (bu == 7).all()
        vs = e.verify_stats()
        assert vs["scanned"] == len(u) and vs["scan_corrupt"] == len(damaged), vs
    finally:
        e.close()


def test_drop_in_counts_a_corrupt_page_as_a_miss(E, gpu, tmp_path, monkeypatch):
    d = tmp_path / "cache"
    d.mkdir()
    u, l, pages, damaged = _corrupt_snapshot(E, 16, str(tmp_path / "good.snap"), str(d / "cachemap_b200.snap"))
    monkeypatch.setenv("CMB200_VERIFY", "1")
    monkeypatch.setenv("CMB200_ARENA_MB", "256")
    cm = E.Cachemap(str(d), 4096, 12, 16)
    assert cm.ok
    try:
        rq0, hit0 = cm.counters()
        for k in range(len(u)):
            got = cm.get(int(l[k]) << 16, 7, 0)
            if k in damaged:
                assert got is None, k
            else:
                assert got == pages[k].tobytes(), k
        rq, hit = cm.counters()
        assert rq - rq0 == len(u) and hit - hit0 == len(u) - len(damaged)
        vs = E.verify_stats(cm.engine_handle())
        assert vs["corrupt"] >= len(damaged)
    finally:
        cm.free()


def test_snapshot_without_fingerprints_reads_unverified(E, gpu, tmp_path):
    u, l, pages, damaged = _corrupt_snapshot(E, 16, str(tmp_path / "good.snap"), str(tmp_path / "nofp.snap"),
                                             with_fp=False)
    ps, flags, recs = snapshot.read_snapshot(str(tmp_path / "good.snap"))
    snapshot.write_snapshot(str(tmp_path / "plain.snap"), ps, recs, with_fingerprints=False)
    e = _engine(E, 16)
    try:
        assert e.load(str(tmp_path / "plain.snap")) == len(u)
        got, st = e.get(u, l)
        assert (st == E.HIT).all() and (got == pages).all()
        got, st = e.get_small(u, l)
        assert (st == E.HIT).all() and (got == pages).all()
        vs = e.verify_stats()
        assert vs["verified"] == 0 and vs["unverified"] == 2 * len(u) and vs["corrupt"] == 0, vs
        _, _, n_bad, checked = e.verify_store()
        assert n_bad == 0 and checked == 0
    finally:
        e.close()


def test_no_false_alarm_under_racing_puts(E, gpu):
    """Readers on their own threads (cmb200_get_small, its own stream) against a writer that alternates
    two contents of the same keys, with compactions and demote / promote rounds in between: a reader
    may stage the old record while the writer publishes the new fingerprint, and must then serve the
    page unverified, never CORRUPT."""
    pshift, count = 16, 32
    n = 1 << pshift
    e = _engine(E, pshift, tier=512 << 20, capacity=512)
    try:
        a = _pages("TM", n, count, 1)
        b = _pages("TR", n, count, 2)
        u, l = _keys(count)
        e.put(u, l, a)
        stop = threading.Event()
        errors = []

        def reader():
            while not stop.is_set():
                got, st = e.get_small(u, l)
                for k in range(count):
                    if st[k] != E.HIT:
                        errors.append(("status", k, int(st[k])))
                    elif not ((got[k] == a[k]).all() or (got[k] == b[k]).all()):
                        errors.append(("torn", k))

        threads = [threading.Thread(target=reader) for _ in range(2)]
        for t in threads:
            t.start()
        try:
            for r in range(60):
                e.put(u, l, b if r % 2 == 0 else a)
                if r % 10 == 3:
                    e.compact()
                if r % 10 == 6:
                    e.demote(u[::3], l[::3])
                if r % 10 == 8:
                    e.promote(u[::3], l[::3])
        finally:
            stop.set()
            for t in threads:
                t.join()
        assert not errors, errors[:10]
        vs = e.verify_stats()
        assert vs["corrupt"] == 0 and vs["verified"] > 0, vs
    finally:
        e.close()


@pytest.mark.parametrize("middle", ["verify", "fingerprint"])
def test_records_without_fingerprints_stay_unverified_across_save_and_load(E, gpu, tmp_path, middle):
    """A record loaded without a fingerprint is saved without one (its slot holds {0, 0} or a fingerprint
    its tag does not name), so the next load serves it unverified and never CORRUPT.  Records put in
    between keep their fingerprints through the same round trip."""
    u, l, pages, _ = _corrupt_snapshot(E, 16, str(tmp_path / "good.snap"), str(tmp_path / "unused.snap"))
    ps, flags, recs = snapshot.read_snapshot(str(tmp_path / "good.snap"))
    snapshot.write_snapshot(str(tmp_path / "plain.snap"), ps, recs, with_fingerprints=False)
    fresh = _pages("TM", 1 << 16, 8, 4242)
    fu, fl = _keys(8, base=1000)
    flags_mid = E.VERIFY if middle == "verify" else E.FINGERPRINT
    e1 = E.Engine(pshift=16, capacity=2048, arena_bytes=256 << 20, flags=flags_mid)
    try:
        assert e1.load(str(tmp_path / "plain.snap")) == len(u)
        e1.put(fu, fl, fresh)
        assert e1.save(str(tmp_path / "again.snap")) == len(u) + 8
    finally:
        e1.close()
    e2 = _engine(E, 16)
    try:
        assert e2.load(str(tmp_path / "again.snap")) == len(u) + 8
        for get in (e2.get, e2.get_small):
            got, st = get(u, l)
            assert (st == E.HIT).all() and (got == pages).all(), get
            got, st = get(fu, fl)
            assert (st == E.HIT).all() and (got == fresh).all(), get
        vs = e2.verify_stats()
        assert vs["corrupt"] == 0 and vs["unverified"] == 2 * len(u) and vs["verified"] == 2 * 8, vs
        _, _, n_bad, checked = e2.verify_store()
        assert n_bad == 0 and checked == 8
    finally:
        e2.close()
