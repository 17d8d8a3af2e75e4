"""GPU tests of cmb200_patch_batch (read-modify-write of stored pages on the device) and of the drop-in
calls over it, cachemap_pread / cachemap_pwrite: a patched page is stored exactly as a put of it would
store it, every status leaves the store as its contract says, a patch is a put and not a get, and no get
ever returns a page's old bytes after a write."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import datagen
import key_edges as K
import snapshot_chain as sc
from ckpt_def import ckpt_words
from oracle import snapshot

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pages(kinds, bs, count, seed):
    return np.stack([datagen.make_page(kinds[i % len(kinds)], bs, seed + i) for i in range(count)])


def _spans(bs, count, rng):
    """Patches (page index, offset, bytes) over `count` pages, in call order: byte 0, the last byte, the
    whole page, single bytes, overlapping spans of one page, and pages named again later in the call."""
    out = [(0, 0, 1), (1, bs - 1, 1), (2, 0, bs)]
    out += [(3, int(o), 1) for o in rng.integers(0, bs, 5)]
    out += [(4, 3, bs // 2), (4, bs // 4, bs // 2), (4, 1, 7), (4, bs // 3, bs - bs // 3)]
    for _ in range(24):
        i = int(rng.integers(0, count))
        n = int(rng.integers(1, 3 if rng.random() < 0.3 else max(2, bs // 3)))
        out.append((i, int(rng.integers(0, bs - n + 1)), n))
    out += [(5, 0, 16), (6, bs // 2 - 1, 2), (count - 1, bs - 17, 17), (5, 8, 16)]   # page 5 again, after others
    return [(i, o, bytes(rng.integers(0, 256, n, dtype=np.uint8))) for i, o, n in out]


def _apply(pages, spans):
    want = pages.copy()
    for i, o, b in spans:
        want[i, o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return want


def _patch(eng, u, l, spans, ts=None):
    idx = np.array([s[0] for s in spans])
    return eng.patch(u[idx], l[idx], [s[1] for s in spans], [s[2] for s in spans],
                     ts=None if ts is None else ts)


def _counters(eng):
    st = eng.stats()
    return st["entries"], st["get_requests"], st["get_hits"], eng.verify_stats()


@pytest.mark.parametrize("accel", [12, 0])
@pytest.mark.parametrize("pshift", [6, 12, 16, 17, 20])
def test_a_patched_page_is_stored_as_a_put_of_it(E, gpu, oracle, tmp_path, pshift, accel):
    bs, count = 1 << pshift, 8
    flags = E.VERIFY if accel else E.FINGERPRINT
    geo = dict(pshift=pshift, accel=accel, capacity=1024, arena_bytes=256 << 20, max_batch=64, flags=flags)
    eng = E.Engine(**geo)
    ref = E.Engine(**geo)
    try:
        pages = _pages("RTZM", bs, count, 300 * pshift + accel)
        u, l = np.full(count, 7, dtype=np.uint64), np.arange(count, dtype=np.uint64)
        eng.put(u, l, pages)
        rng = np.random.default_rng(pshift * 10 + accel)
        spans = _spans(bs, count, rng)
        ts = np.arange(1000, 1000 + len(spans), dtype=np.uint64)
        before, chunks = _counters(eng), eng.stats()["put_chunks"]
        st = _patch(eng, u, l, spans, ts)
        assert (st == E.HIT).all(), st
        assert _counters(eng) == before                      # not a get: no request, hit or verification
        assert eng.stats()["put_chunks"] == chunks + count   # one stored page per address
        want = _apply(pages, spans)
        # the records: byte for byte what the reference stores for the patched page
        model = oracle.StoreModel(pshift, accel)
        for i in range(count):
            model.put(*K.cachemap_args(7, i, pshift), want[i])
        recs = eng.read_records(u, l)
        for i in range(count):
            assert recs[i] == model.record_bytes(7, i), i
        got, gs = eng.get(u, l)
        assert (gs == E.HIT).all() and (got == want).all()
        if pshift <= 17:
            got, gs = eng.get_small(u, l)
            assert (gs == E.HIT).all() and (got == want).all()
        fps, ok = eng.read_fingerprints(u, l)
        assert ok.all() and (fps == E.fingerprint_batch(want)).all()
        # fingerprint and parse checkpoints as a put of the patched pages leaves them
        ref.put(u, l, want)
        rw, rok = ref.read_checkpoints(u, l)
        w, wok = eng.read_checkpoints(u, l)
        assert (wok == rok).all(), (wok, rok)
        for i in range(count):
            if wok[i] == 1:
                assert w[i, 1:].tolist() == rw[i, 1:].tolist() == ckpt_words(recs[i][24:], bs)[1:], i
        # ts of the last patch of each page, in the snapshot the store writes
        last = {}
        for k, (i, _o, _b) in enumerate(spans):
            last[i] = int(ts[k])
        eng.save(str(tmp_path / "s.snap"))
        saved = {sc.addr_of(r[3])[1]: r[0] for r in snapshot.read_snapshot(str(tmp_path / "s.snap"))[2]}
        assert saved == last
    finally:
        eng.close()
        ref.close()


def test_statuses_of_absent_and_key_sharing_addresses(E, gpu, oracle):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=64)
    try:
        u, l = np.full(4, 3, dtype=np.uint64), np.arange(4, dtype=np.uint64)
        eng.put(u[:2], l[:2], _pages("RT", bs, 2, 5))
        st = eng.patch(u[2:], l[2:], [0, 100], [b"x", b"yz"])
        assert (st == E.MISS).all() and eng.entries() == 2
        _, gs = eng.get(u[2:], l[2:])
        assert (gs == E.MISS).all()
        fx = K.load()
        for name in ("quad", "pair0", "key0", "key_ones"):
            a, other = fx["groups"][name][:2]
            page = _pages("M", bs, 1, 40)
            ou, ol = np.array([other[0]], dtype=np.uint64), np.array([other[1]], dtype=np.uint64)
            eng.put(ou, ol, page)
            rec = eng.read_records(ou, ol)[0]
            st = eng.patch(np.array([a[0]], dtype=np.uint64), np.array([a[1]], dtype=np.uint64), [5], [b"abc"])
            assert st.tolist() == [E.BAD_ENTRY], name
            assert eng.read_records(ou, ol)[0] == rec, name
            got, gs = eng.get(ou, ol)
            assert gs[0] == E.HIT and (got[0] == page[0]).all(), name
        # out-of-page extents and empty patches are refused before anything is applied
        rec0 = eng.read_records(u[:1], l[:1])[0]
        for off, data in ((bs - 1, b"ab"), (0, b""), (bs, b"a")):
            with pytest.raises(RuntimeError):
                eng.patch(np.array([3, 3], dtype=np.uint64), np.array([0, 1], dtype=np.uint64), [0, off], [b"q", data])
        assert eng.read_records(u[:1], l[:1])[0] == rec0
    finally:
        eng.close()


def test_an_untrusted_record_is_removed(E, gpu, oracle, tmp_path):
    """A snapshot whose second record carries a fingerprint its page does not have: under CMB200_VERIFY
    the patch answers CORRUPT and the key is gone; the clean record is patched."""
    pshift, bs = 12, 4096
    pages = _pages("TR", bs, 2, 77)
    model = oracle.StoreModel(pshift, 12)
    recs = []
    for i in range(2):
        model.put(*K.cachemap_args(9, i, pshift), pages[i])
        hi, lo = oracle.fingerprint128(pages[i])
        recs.append((50 + i, hi, lo ^ (i == 1), model.record_bytes(9, i)))
    path = str(tmp_path / "bad.snap")
    snapshot.write_snapshot(path, pshift, recs, with_fingerprints=True)
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.VERIFY)
    try:
        assert eng.load(path) == 2
        u, l = np.full(2, 9, dtype=np.uint64), np.arange(2, dtype=np.uint64)
        st = eng.patch(u, l, [10, 10], [b"hello", b"hello"])
        assert st.tolist() == [E.HIT, E.CORRUPT]
        assert eng.entries() == 1
        got, gs = eng.get(u, l)
        want = pages[0].copy()
        want[10:15] = np.frombuffer(b"hello", dtype=np.uint8)
        assert gs.tolist() == [E.HIT, E.MISS] and (got[0] == want).all()
        assert eng.verify_stats()["corrupt"] == 0           # the patch's decode is not a get
    finally:
        eng.close()


def test_a_full_arena_drops_the_old_page(E, gpu):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=1 << 20, max_batch=64)
    try:
        n = 320                                              # incompressible: more than 1 MiB of records
        pages = _pages("R", bs, n, 11)
        u, l = np.full(n, 4, dtype=np.uint64), np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        assert eng.stats()["dropped_puts"] > 0
        _, gs = eng.get(u, l)
        live = np.flatnonzero(gs == E.HIT)[:3]
        entries = eng.entries()
        st = eng.patch(u[live], l[live], [0, 1, 2], [b"a", b"b", b"c"])
        assert (st == E.DROPPED).all(), st
        _, gs = eng.get(u[live], l[live])
        assert (gs == E.MISS).all() and eng.entries() == entries - 3
    finally:
        eng.close()


def test_a_host_tier_record_comes_back_patched(E, gpu, oracle):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64,
                   host_tier_bytes=8 << 20, flags=E.FINGERPRINT)
    try:
        count = 16
        pages = _pages("RTZM", bs, count, 21)
        u, l = np.full(count, 6, dtype=np.uint64), np.arange(count, dtype=np.uint64)
        eng.put(u, l, pages)
        assert eng.demote(u, l) == count
        old = eng.read_records(u[:4], l[:4])
        ht0, hot0 = eng.host_tier_stats(), eng.tier_hot()
        st = eng.patch(u[:4], l[:4], [0, 17, 100, bs - 3], [b"A", b"BB", b"C" * 200, b"DDD"])
        assert (st == E.HIT).all()
        ht1 = eng.host_tier_stats()
        assert ht1["records"] == ht0["records"] - 4 and ht1["hits"] == ht0["hits"]
        assert ht1["garbage"] >= ht0["garbage"] + sum(len(r) for r in old)
        assert len(eng.tier_hot()[0]) == 0 and len(hot0[0]) == 0
        want = _apply(pages, [(0, 0, b"A"), (1, 17, b"BB"), (2, 100, b"C" * 200), (3, bs - 3, b"DDD")])
        model = oracle.StoreModel(pshift, 12)
        for i in range(4):
            model.put(*K.cachemap_args(6, i, pshift), want[i])
        assert eng.read_records(u[:4], l[:4]) == [model.record_bytes(6, i) for i in range(4)]
        got, gs = eng.get(u, l)
        assert (gs == E.HIT).all() and (got == want).all()
        assert eng.host_tier_stats()["hits"] == ht1["hits"] + count - 4   # the patched pages are in the arena
    finally:
        eng.close()


def test_a_chain_delta_holds_the_patch(E, gpu, tmp_path):
    pshift, bs = 12, 4096
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.FINGERPRINT)
    eng = E.Engine(**geo)
    try:
        count = 24
        pages = _pages("RTZM", bs, count, 31)
        u, l = np.full(count, 8, dtype=np.uint64), np.arange(count, dtype=np.uint64)
        eng.put(u, l, pages)
        base = str(tmp_path / "c.snap")
        E.snapshot_finish(E.chain_begin([eng.h], base, False))
        assert (eng.patch(u[[3, 9]], l[[3, 9]], [5, 4000], [b"xyz", b"q" * 96]) == E.HIT).all()
        E.snapshot_finish(E.chain_begin([eng.h], base, True))
        d = sc.read_delta(base + ".d1")
        assert d["tombstones"] == [] and sorted(sc.addr_of(r[3]) for r in d["records"]) == [(8, 3), (8, 9)]
        want = _apply(pages, [(3, 5, b"xyz"), (9, 4000, b"q" * 96)])
        e2 = E.Engine(**geo)
        try:
            assert E.load_chain([e2.h], base) == (count, 1)
            got, gs = e2.get(u, l)
            assert (gs == E.HIT).all() and (got == want).all()
        finally:
            e2.close()
    finally:
        eng.close()


def test_refused_after_a_multi_gpu_call(E, gpu):
    eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64)
    try:
        one = np.array([1], dtype=np.uint64)
        eng.put(one, one, _pages("R", 4096, 1, 1))
        assert eng.patch(one, one, [0], [b"a"]).tolist() == [E.HIT]
        eng.set_stream_order(100, 2)
        with pytest.raises(RuntimeError, match="multi-GPU"):
            eng.patch(one, one, [0], [b"b"])
    finally:
        eng.close()


def test_small_gets_during_patches_see_old_or_new_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 96, 65536
eng = E.Engine(pshift=16, accel=12, capacity=4096, arena_bytes=2 << 30, max_batch=256)
A = np.stack([E.gen_chunk_host(7, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(7, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 55, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
eng.put(u, l, A)
stop = threading.Event(); bad = []
def reader():
    while not stop.is_set():
        out, st = eng.get_small(u, l)
        ok = (st == E.HIT) & ((out == A).all(axis=1) | (out == B).all(axis=1))
        if not ok.all():
            bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
            return
th = [threading.Thread(target=reader) for _ in range(2)]
[t.start() for t in th]
for rnd in range(30):
    src = B if rnd % 2 == 0 else A
    # each page in three spans of one call: a reader that saw a part of them would see a mix
    cut = [0, 20000, 45000, bs]
    uu = np.repeat(u, 3); ll = np.repeat(l, 3)
    offs = [cut[k] for _ in range(n) for k in range(3)]
    data = [src[i, cut[k]:cut[k + 1]].tobytes() for i in range(n) for k in range(3)]
    assert (eng.patch(uu, ll, offs, data) == E.HIT).all()
stop.set(); [t.join() for t in th]
assert not bad, bad
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
print("no mixed pages")
'''
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no mixed pages" in out.stdout, out.stdout + out.stderr


DROP_IN = textwrap.dedent("""
    import os, pickle, shutil, sys, threading, time
    sys.path.insert(0, sys.argv[1])
    import numpy as np
    import edge_fuse_b200 as E
    d, seed, ps, N, mode, phase = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sys.argv[6], sys.argv[7]
    P = 1 << ps                                           # N pages per object
    objs = (3, 4, 5)
    fails = []

    def check(what, cond):
        if not cond:
            fails.append(what)

    if phase == "read":                                   # a second process opens what the first one left
        with open(d + ".model", "rb") as f:
            model, cached = pickle.load(f)
        cm = E.Cachemap(d, 1 << 16, 12, ps)
        assert cm.ok
        for o in objs:
            for p in range(N):
                g = cm.get(p * P, o, 0)
                check(("restart get", o, p), (g is not None) == (p in cached[o]))
                check(("restart stale", o, p), g is None or g == bytes(model[o][p * P:(p + 1) * P]))
        cm.free()
        print("fails", len(fails), fails[:5])
        sys.exit(0)

    # exact: every page the model caches hits and no other does; evict: the capacity is below the
    # working set, so only "never stale" holds, and pread returns bytes exactly when every page of its
    # range hits; stale: the flusher drops pages in the background, so only "never stale" holds;
    # restart: exact, then the directory is copied as a crash leaves it for the read phase
    exact = mode in ("exact", "restart")
    cm = E.Cachemap(d, 1024 if mode == "evict" else 1 << 16, 12, ps)
    assert cm.ok
    rng = np.random.default_rng(seed)
    model = {o: bytearray(rng.integers(0, 256, N * P, dtype=np.uint8).tobytes()) for o in objs}
    cached = {o: set() for o in objs}
    for o in objs:                                        # most pages cached whole, a few not
        for p in range(N):
            if rng.random() < 0.8:
                cm.write_range(o, 0, p * P, bytes(model[o][p * P:(p + 1) * P]))
                cached[o].add(p)

    def want_read(o, off, size):
        pages = range(off // P, (off + size - 1) // P + 1) if size else []
        rq = ht = 0
        for p in pages:
            rq += 1
            if p not in cached[o]:
                return False, rq, ht
            ht += 1
        return True, rq, ht

    def rand_range():
        kind = rng.integers(0, 4)
        if kind == 0:                                     # inside one page
            p = int(rng.integers(0, N)); a = int(rng.integers(0, P)); b = int(rng.integers(a + 1, P + 1))
            return p * P + a, b - a
        if kind == 1:                                     # many pages, ragged ends
            a = int(rng.integers(0, (N - 8) * P)); return a, int(rng.integers(P, 8 * P))
        if kind == 2:                                     # aligned
            p = int(rng.integers(0, N - 4)); return p * P, int(rng.integers(1, 5)) * P
        a = int(rng.integers(1, N * P - 3)); return a, int(rng.integers(1, min(3 * P, N * P - a)))

    def pwrite(o, off, size):
        data = rng.integers(0, 256, size, dtype=np.uint8).tobytes()
        cm.pwrite(o, 0, off, data)
        model[o][off:off + size] = data
        first, last = off // P, (off + size - 1) // P
        for p in range(first, last + 1):
            if p * P >= off and (p + 1) * P <= off + size:
                cached[o].add(p)                          # covered whole: put

    def sweep():                                          # every page: hit with the model's bytes, or miss
        for oo in objs:
            for p in range(N):
                g = cm.get(p * P, oo, 0)
                check(("get", oo, p, g is not None), not exact or (g is not None) == (p in cached[oo]))
                check(("stale", oo, p), g is None or g == bytes(model[oo][p * P:(p + 1) * P]))

    for step in range(400):
        o = objs[int(rng.integers(0, len(objs)))]
        off, size = rand_range()
        if rng.random() < 0.5:
            pwrite(o, off, size)
        else:
            r0 = cm.counters()
            got = cm.pread(o, 0, off, size)
            r1 = cm.counters()
            check(("bytes", o, off, size), got is None or got == bytes(model[o][off:off + size]))
            if exact:
                ok, rq, ht = want_read(o, off, size)
                check(("pread", o, off, size, ok, got is not None), (got is not None) == ok)
                check(("counters", o, off, size), (r1[0] - r0[0], r1[1] - r0[1]) == (rq, ht))
            elif mode == "evict":                         # bytes exactly when every page of the range hits now
                every = all(cm.get(p * P, o, 0) is not None for p in range(off // P, (off + size - 1) // P + 1))
                check(("pread", o, off, size, every, got is not None), (got is not None) == every)
            if off % P == 0 and size % P == 0 and exact:  # aligned: exactly read_range
                r2 = cm.counters()
                alt = cm.read_range(o, 0, off, size)
                r3 = cm.counters()
                check(("aligned", o, off, size), alt == got and (r3[0] - r2[0], r3[1] - r2[1]) == (rq, ht))
        if step % 50 == 49:
            sweep()

    if mode == "restart":
        # the write-behind ring drains (engine_handles waits for it) and a base is written, so that the
        # next tick writes a delta; then unaligned writes over cached pages, whose edge pages are patched
        # by the engine, and the store left until that tick has written them
        cm.engine_handles()
        check("a base written", cm.checkpoint() == 0)
        for k in range(12):
            o = objs[k % 3]
            p = sorted(cached[o])[(7 * k) % len(cached[o])]
            pwrite(o, p * P + 1 + k, P - 2 - k)
            if p + 1 < N:
                pwrite(o, p * P + P // 2, P)              # the end of p and the start of p + 1
        sweep()
        names = lambda: sorted((f, os.stat(os.path.join(d, f)).st_mtime_ns) for f in os.listdir(d))
        seen, quiet, t0 = names(), time.time(), time.time()
        while time.time() - quiet < 3.5 and time.time() - t0 < 60:      # no tick for more than 3 ticks
            time.sleep(0.1)
            now = names()
            if now != seen:
                seen, quiet = now, time.time()
        copy = d + ".copy"
        shutil.copytree(d, copy)                          # the directory as a crash leaves it
        with open(copy + ".model", "wb") as f:
            pickle.dump((model, cached), f)
        print("files", " ".join(f for f, _ in seen), flush=True)
        print("fails", len(fails), fails[:5], flush=True)
        os._exit(0)

    # 16 threads write disjoint bytes of one cached page: every write lands
    cm.write_range(9, 0, 0, bytes(P))
    last = [None] * 16

    def writer(t):
        r = np.random.default_rng(100 + t)
        for k in range(40):
            b = r.integers(0, 256, 40, dtype=np.uint8).tobytes()
            cm.pwrite(9, 0, 7 + 40 * t, b)
            last[t] = b
    th = [threading.Thread(target=writer, args=(t,)) for t in range(16)]
    [t.start() for t in th]
    [t.join() for t in th]
    page = cm.pread(9, 0, 0, P)
    check("threads page", page is not None or not exact)
    for t in range(16):
        check(("thread", t), page is None or page[7 + 40 * t:47 + 40 * t] == last[t])
    cm.free()
    print("fails", len(fails), fails[:5])
""")

# (environment, page shift, pages per object, mode); every case drives the byte model above
DROP_IN_CASES = {
    "ring": ({}, 12, 48, "exact"),
    "no_ring": ({"CMB200_WB_SLOTS": "0"}, 12, 48, "exact"),
    "two_engines": ({"CMB200_DEVICES": "0,0"}, 12, 48, "exact"),
    # 128 KiB pages: pread's edge pages decode in the fused pair kernel
    "pshift17": ({}, 17, 48, "exact"),
    # 1 MiB pages: no fused get, and records that leave the arena check no margin
    "pshift20": ({}, 20, 12, "exact"),
    # 3 MiB of incompressible pages over a 1 MiB arena: writes demote, reads promote, and pwrite
    # patches host-tier records after filemap_arena_room has made room.  A ring of 64 slots flushes
    # batches that demotion always makes room for
    "host_tier": ({"CMB200_ARENA_MB": "1", "CMB200_HOST_TIER_MB": "64", "CMB200_TIER_PROMOTE": "1",
                   "CMB200_WB_SLOTS": "64"}, 12, 256, "exact"),
    # the default ring flushes batches larger than the whole arena: pages are dropped, never stale
    "host_tier_full_batches": ({"CMB200_ARENA_MB": "1", "CMB200_HOST_TIER_MB": "64", "CMB200_TIER_PROMOTE": "1"},
                               12, 256, "stale"),
    "verify_evict_access": ({"CMB200_VERIFY": "1", "CMB200_EVICT": "access"}, 12, 48, "exact"),
    # 1 024 pages (the least capacity a map accepts) for 3 x 512: eviction runs; synchronous puts, so
    # that nothing evicts between a pread and the gets that check it
    "evict": ({"CMB200_WB_SLOTS": "0"}, 12, 512, "evict"),
    "evict_access": ({"CMB200_WB_SLOTS": "0", "CMB200_EVICT": "access"}, 14, 512, "evict"),
    "restart": ({"CMB200_PERSIST": "1", "CMB200_CHECKPOINT_SEC": "1", "CMB200_CHECKPOINT_DELTAS": "64"}, 12, 48,
                "restart"),
}


@pytest.mark.parametrize("case", list(DROP_IN_CASES))
def test_drop_in_pread_pwrite_match_a_model(E, gpu, tmp_path, case):
    env, ps, n, mode = DROP_IN_CASES[case]
    script = tmp_path / "drive.py"
    script.write_text(DROP_IN)
    base = dict(os.environ, CMB200_PERSIST="0", CMB200_ARENA_MB="256")
    for k in ("CMB200_DEVICES", "CMB200_WB_SLOTS", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_VERIFY", "CMB200_EVICT"):
        base.pop(k, None)
    base.update(env)
    d = tmp_path / "cache"
    d.mkdir()
    args = [sys.executable, str(script), ROOT, str(d), "17", str(ps), str(n), mode]
    r = subprocess.run(args + ["run"], capture_output=True, text=True, timeout=600, env=base)
    assert r.returncode == 0 and "fails 0 []" in r.stdout, r.stdout + r.stderr[-3000:]
    if mode == "restart":
        assert ".d1" in r.stdout.split("files", 1)[1], r.stdout      # the tick wrote a delta
        args[3] = str(d) + ".copy"
        r = subprocess.run(args + ["read"], capture_output=True, text=True, timeout=600, env=base)
        assert r.returncode == 0 and "fails 0 []" in r.stdout, r.stdout + r.stderr[-3000:]
