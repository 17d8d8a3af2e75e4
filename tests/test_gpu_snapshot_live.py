"""GPU tests of the live snapshot (cmb200_snapshot_begin / _finish): the engines are locked only while
their live records are listed, the records are written while the engines keep serving, and the file is
the store as it was at begin — whatever puts, unsets, demotions, promotions, compactions and host-tier
laps happen while it is written."""
import collections
import os
import shutil
import threading
import time

import numpy as np
import pytest

import datagen
from oracle import snapshot

pytestmark = pytest.mark.gpu

NH = 5


def _addrs(oracle, offs, pshift):
    ul = [oracle.addr_compose(int(o), NH, 0, pshift) for o in offs]
    return (np.array([a[0] for a in ul], dtype=np.uint64), np.array([a[1] for a in ul], dtype=np.uint64))


def _multiset(path):
    return collections.Counter(snapshot.read_snapshot(path)[2])


class _Store:
    """An engine, its oracle.StoreModel and the page of every live key, changed together."""

    def __init__(self, E, oracle, eng, pshift, accel):
        self.E, self.oracle, self.eng, self.pshift = E, oracle, eng, pshift
        self.model = oracle.StoreModel(pshift, accel)
        self.pages = {}
        self.ts = 1

    def put(self, idx, pages):
        u, l = _addrs(self.oracle, [i << self.pshift for i in idx], self.pshift)
        ts = np.arange(self.ts, self.ts + len(idx), dtype=np.uint64)
        self.ts += len(idx)
        self.eng.put(u, l, pages, ts=ts)
        for i, p in zip(idx, pages):
            self.model.put(i << self.pshift, NH, 0, p)
            self.pages[i] = p

    def unset(self, idx):
        u, l = _addrs(self.oracle, [i << self.pshift for i in idx], self.pshift)
        self.eng.unset(u, l)
        for i, a, b in zip(idx, u, l):
            self.model.unset(int(a), int(b))
            del self.pages[i]

    def addrs(self, idx):
        return _addrs(self.oracle, [i << self.pshift for i in idx], self.pshift)

    def records(self):
        """The model's record bytes of every live key."""
        idx = sorted(self.pages)
        u, l = self.addrs(idx)
        return sorted(self.model.record_bytes(int(a), int(b)) for a, b in zip(u, l))


def _serves(E, eng, oracle, pshift, pages):
    idx = sorted(pages)
    u, l = _addrs(oracle, [i << pshift for i in idx], pshift)
    want = np.stack([pages[i] for i in idx])
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st == E.HIT).all() and (out == want).all()


@pytest.mark.parametrize("pshift", [12, 16, 17])
@pytest.mark.parametrize("accel", [12, 0])
def test_file_is_the_store_at_begin(E, gpu, oracle, tmp_path, pshift, accel):
    bs, n = 1 << pshift, 96
    geo = dict(pshift=pshift, accel=accel, capacity=4096, arena_bytes=256 << 20, max_batch=64, flags=E.FINGERPRINT)
    eng = E.Engine(host_tier_bytes=64 << 20, **geo)
    s = _Store(E, oracle, eng, pshift, accel)
    kinds = "RTZMPAXS"
    s.put(list(range(n)), np.stack([datagen.make_page(kinds[i % 8], bs, 40 + i) for i in range(n)]))
    s.put(list(range(0, n, 6)), np.stack([datagen.make_page(kinds[(i + 3) % 8], bs, 900 + i) for i in range(0, n, 6)]))
    tier_keys = list(range(1, 25, 3))
    u, l = s.addrs(tier_keys)
    assert eng.demote(u, l) == len(tier_keys)
    ref = str(tmp_path / "ref.snap")
    path = str(tmp_path / "live.snap")
    assert eng.save(ref) == n
    at_begin_pages, at_begin_records = dict(s.pages), s.records()

    h = eng.snapshot_begin(path)
    s.put(list(range(n, n + 16)), np.stack([datagen.make_page(kinds[i % 8], bs, 2000 + i) for i in range(16)]))
    s.put(list(range(2, 50, 6)), np.stack([datagen.make_page("T", bs, 3000 + i) for i in range(2, 50, 6)]))
    s.unset(list(range(5, 60, 7)))
    u, l = s.addrs(list(range(60, 90, 4)))
    assert eng.demote(u, l) > 0
    u, l = s.addrs(tier_keys)
    assert eng.promote(u, l) > 0
    eng.compact()
    s.put(list(range(n + 16, n + 24)), np.stack([datagen.make_page("M", bs, 4000 + i) for i in range(8)]))
    assert E.snapshot_finish(h) == n

    # a quiescent store at begin: the same bytes as a save at that moment
    assert open(path, "rb").read() == open(ref, "rb").read()
    got = snapshot.read_snapshot(path)[2]
    assert collections.Counter(got) == _multiset(ref)
    assert sorted(r[3] for r in got) == at_begin_records
    e2 = E.Engine(**geo)
    assert e2.load(path) == n and e2.entries() == n
    _serves(E, e2, oracle, pshift, at_begin_pages)
    e2.close()
    assert eng.entries() == len(s.pages)
    _serves(E, eng, oracle, pshift, s.pages)
    eng.close()


def test_tier_laps_during_a_snapshot(E, gpu, tmp_path):
    pshift, bs, n = 12, 4096, 300
    geo = dict(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128,
               host_tier_bytes=256 << 10)                      # ~62 incompressible records per lap
    pages = np.stack([datagen.make_page("R", bs, 700 + i) for i in range(n)])
    u = np.full(n, 6, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    eng, twin = E.Engine(**geo), E.Engine(**geo)
    for e in (eng, twin):
        e.put(u, l, pages)
        assert e.demote(u[:50], l[:50]) == 50
    tier_recs = eng.read_records(u[:50], l[:50])
    ref = str(tmp_path / "ref.snap")
    path = str(tmp_path / "live.snap")
    assert eng.save(ref) == n
    h = eng.snapshot_begin(path)
    for e in (eng, twin):
        for base in range(50, n, 50):                          # four laps of the tier
            assert e.demote(u[base:base + 50], l[base:base + 50]) == 50
    assert E.snapshot_finish(h) == n
    assert open(path, "rb").read() == open(ref, "rb").read()
    in_file = {r[3] for r in snapshot.read_snapshot(path)[2]}
    assert all(r in in_file for r in tier_recs)                # the pre-begin tier, byte for byte
    e2 = E.Engine(**dict(geo, host_tier_bytes=0))
    assert e2.load(path) == n
    out, st = e2.get(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    e2.close()
    ht, hw = eng.host_tier_stats(), twin.host_tier_stats()
    assert ht["retired_records"] > 0
    assert ht["retired_records"] == hw["retired_records"] and eng.entries() == twin.entries()
    for fn in ("get", "get_small"):
        (o1, s1), (o2, s2) = getattr(eng, fn)(u, l), getattr(twin, fn)(u, l)
        assert (s1 == s2).all() and (o1[s1 == E.HIT] == pages[s1 == E.HIT]).all()
    eng.close()
    twin.close()


def test_several_engines(E, gpu, oracle, tmp_path):
    pshift, bs, n = 16, 65536, 256
    geo = dict(pshift=pshift, accel=12, capacity=4096, arena_bytes=256 << 20, max_batch=128, device=0)
    engs = [E.Engine(**geo), E.Engine(**geo)]
    u, l = _addrs(oracle, [i << pshift for i in range(n + 64)], pshift)
    own = np.array([E.owner(oracle.addr_key(int(a), int(b)), 2) for a, b in zip(u, l)])
    pages = np.stack([datagen.make_page("RTZMPAX"[i % 7], bs, 60 + i) for i in range(n + 64)])
    for k in (0, 1):
        sel = np.nonzero(own[:n] == k)[0]
        engs[k].put(u[sel], l[sel], pages[sel])
    path = str(tmp_path / "set.snap")
    h = E.snapshot_begin([e.h for e in engs], path)
    newer = np.stack([datagen.make_page("T", bs, 5000 + i) for i in range(n)])
    for k in (0, 1):
        sel = np.nonzero(own[:n] == k)[0]
        engs[k].put(u[sel[:20]], l[sel[:20]], newer[sel[:20]])
        engs[k].unset(u[sel[20:40]], l[sel[20:40]])
        extra = n + np.nonzero(own[n:] == k)[0]
        engs[k].put(u[extra], l[extra], pages[extra])
        engs[k].compact()
    assert E.snapshot_finish(h) == n
    for g in (1, 3):
        fresh = [E.Engine(**geo) for _ in range(g)]
        assert E.load_set([e.h for e in fresh], path) == n
        assert sum(e.entries() for e in fresh) == n
        own_g = np.array([E.owner(oracle.addr_key(int(a), int(b)), g) for a, b in zip(u[:n], l[:n])])
        for k, e in enumerate(fresh):
            sel = np.nonzero(own_g == k)[0]
            out, st = e.get(u[sel], l[sel])
            assert (st == E.HIT).all() and (out == pages[sel]).all(), (g, k)
            out, st = e.get(u[n:], l[n:])
            assert (st == E.MISS).all()
            e.close()
    for e in engs:
        e.close()


def _page(bs, key, ver):
    w = np.arange(bs // 8, dtype=np.uint64)
    w += np.full(1, key, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(ver << 20)   # wraps mod 2^64
    w[1::4] = np.uint64(ver)                                   # compressible, and the version is in plain sight
    return w.view(np.uint8)


def _page_version(page, key):
    """Version of a well-formed page of `key`, or -1 (torn or somebody else's)."""
    bs = len(page)
    ver = int(page.view(np.uint64)[1])
    return ver if (page == _page(bs, key, ver)).all() else -1


def test_concurrent_puts_and_gets_during_snapshots(E, gpu, tmp_path):
    pshift, bs, keys = 12, 4096, 3072
    eng = E.Engine(pshift=pshift, accel=12, capacity=16384, arena_bytes=256 << 20, max_batch=256, flags=E.VERIFY)
    u = np.full(keys, 9, dtype=np.uint64)
    l = np.arange(keys, dtype=np.uint64)
    done_ver = {}                                              # key -> newest version whose put returned
    first_issued = []                                          # keys in the order of their first put
    stop = threading.Event()
    errors = []

    def worker():
        rng = np.random.default_rng(3)
        ver = np.zeros(keys, dtype=np.int64)
        nxt = 0
        while not stop.is_set():
            if nxt < keys and (nxt < 256 or rng.random() < 0.5):
                idx = np.arange(nxt, min(nxt + 64, keys))
                first_issued.extend(idx.tolist())
                nxt += len(idx)
            else:
                idx = np.unique(rng.integers(0, nxt, 64))
            ver[idx] += 1
            eng.put(u[idx], l[idx], np.stack([_page(bs, int(k), int(ver[k])) for k in idx]))
            for k in idx:
                done_ver[int(k)] = int(ver[k])
            q = rng.integers(0, nxt, 32)
            out, st = eng.get_small(u[q], l[q])
            for j, k in enumerate(q):
                if st[j] != E.HIT or _page_version(out[j], int(k)) < 1:
                    errors.append(("get", int(k), int(st[j])))

    th = threading.Thread(target=worker)
    th.start()
    cycles = []
    try:
        for c in range(4):
            time.sleep(0.3)
            before = dict(done_ver)
            path = str(tmp_path / f"c{c}.snap")
            h = eng.snapshot_begin(path)
            issued = set(first_issued)
            time.sleep(0.1)
            E.snapshot_finish(h)
            cycles.append((path, before, issued))
    finally:
        stop.set()
        th.join()
    assert not errors, errors[:8]
    for path, before, issued in cycles:
        recs = snapshot.read_snapshot(path)[2]
        in_file = {int(np.frombuffer(r[3][8:16], dtype=np.uint64)[0]) for r in recs}
        assert set(before) <= in_file, path
        assert in_file <= issued, path
        e2 = E.Engine(pshift=pshift, accel=12, capacity=16384, arena_bytes=256 << 20, max_batch=256, flags=E.VERIFY)
        assert e2.load(path) == len(recs) == len(in_file)
        ks = np.array(sorted(in_file), dtype=np.uint64)
        out, st = e2.get(u[ks], l[ks])
        assert (st == E.HIT).all(), np.unique(st)
        for j, k in enumerate(ks):
            v = _page_version(out[j], int(k))
            assert v >= before.get(int(k), 1), (path, int(k), v, before.get(int(k)))
        assert e2.verify_store()[2] == 0 and e2.verify_stats()["corrupt"] == 0
        e2.close()
    eng.close()


def test_drop_in_checkpoints_while_puts_run(E, gpu, tmp_path, monkeypatch):
    monkeypatch.setenv("CMB200_CHECKPOINT_SEC", "1")
    monkeypatch.setenv("CMB200_PERSIST", "1")
    for k in ("CMB200_DEVICES", "CMB200_HOST_TIER_MB", "CMB200_ARENA_MB"):
        monkeypatch.delenv(k, raising=False)
    pshift, bs, keys = 12, 4096, 2048
    d = tmp_path / "cache"
    d.mkdir()
    snap = str(d / "cachemap_b200.snap")
    cm = E.Cachemap(str(d), 16384, 12, pshift)
    assert cm.ok
    last = {}
    stop = threading.Event()

    def putter():
        ver = 0
        while not stop.is_set():
            ver += 1
            for k in range(0, keys, 7):
                kk = (k + ver) % keys
                cm.put(kk << pshift, 3, 0, _page(bs, kk, ver))
                last[kk] = ver
                if stop.is_set():
                    break

    th = threading.Thread(target=putter)
    th.start()
    seen, parsed = set(), 0
    t_end = time.time() + 4.0
    try:
        while time.time() < t_end:
            try:
                st = os.stat(snap)
            except FileNotFoundError:
                time.sleep(0.02)
                continue
            if st.st_ino not in seen:
                seen.add(st.st_ino)
                copy = str(tmp_path / f"copy{len(seen)}.snap")
                shutil.copyfile(snap, copy)
                snapshot.read_snapshot(copy)
                parsed += 1
            time.sleep(0.02)
    finally:
        stop.set()
        th.join()
    assert len(seen) >= 2 and parsed == len(seen), (len(seen), parsed)
    cm.free()
    cm2 = E.Cachemap(str(d), 16384, 12, pshift)
    for kk, ver in last.items():
        got = cm2.get(kk << pshift, 3, 0)
        assert got is not None and _page_version(np.frombuffer(got, dtype=np.uint8).copy(), kk) == ver, kk
    cm2.free()


def test_errors_and_a_second_begin(E, gpu, tmp_path):
    missing = tmp_path / "no" / "such"
    eng = E.Engine(pshift=16, accel=0, capacity=16384, arena_bytes=1 << 30, max_batch=512)
    with pytest.raises(RuntimeError):
        eng.snapshot_begin(str(missing / "x.snap"))
    assert not (tmp_path / "no").exists() and os.listdir(tmp_path) == []
    # a store of 512 MiB of raw pages takes a while to write: a second begin waits for the first one
    n, bs = 8192, 65536
    for base in range(0, n, 512):
        idx = np.arange(base, base + 512, dtype=np.uint64)
        eng.put(np.full(512, 4, dtype=np.uint64), idx, np.stack([datagen.make_page("R", bs, int(i)) for i in idx]))
    p1, p2 = str(tmp_path / "a.snap"), str(tmp_path / "b.snap")
    h1 = eng.snapshot_begin(p1)
    t = {}

    def second():
        t["call"] = time.perf_counter()
        t["h"] = eng.snapshot_begin(p2)
        t["ret"] = time.perf_counter()

    th = threading.Thread(target=second)
    th.start()
    assert E.snapshot_finish(h1) == n
    t_finish1 = time.perf_counter()
    th.join()
    assert E.snapshot_finish(t["h"]) == n
    assert t["call"] < t_finish1 - 0.05, t                     # the second begin was called while the first wrote
    assert t["ret"] > t_finish1 - 0.05, t                      # and returned only once that was written
    assert open(p1, "rb").read() == open(p2, "rb").read()
    assert sorted(os.listdir(tmp_path)) == ["a.snap", "b.snap"]
    eng.close()
