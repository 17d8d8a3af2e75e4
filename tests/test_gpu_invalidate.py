"""GPU tests of cmb200_invalidate and cachemap_invalidate: every live record whose stored address is
{u, l} with l in an interval goes, through either kernel (k_invalidate_keys for a short interval,
k_invalidate_scan for a long one), and nothing else does: not another generation of the object, not
another object's page that shares a key.  Checked against a store model, through the host tier,
snapshots and chains, verified gets, concurrent small gets, the table rebuild, and the drop-in over
two engines."""
import os
import shutil
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

TO_END = (1 << 64) - 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ua(addrs):
    return (np.array([a[0] for a in addrs], dtype=np.uint64), np.array([a[1] for a in addrs], dtype=np.uint64))


def _pages(bs, n, seed):
    kinds = "RTZMPAXS"
    return np.stack([datagen.make_page(kinds[(seed + i) % 8], bs, seed * 131 + i) for i in range(n)])


class Model:
    """oracle.StoreModel with invalidation by stored address; addresses are (u, l) pairs."""

    def __init__(self, oracle, pshift, accel=12):
        self.O, self.pshift = oracle, pshift
        self.m = oracle.StoreModel(pshift, accel)

    def put(self, addrs, pages):
        for a, p in zip(addrs, pages):
            self.m.put(*K.cachemap_args(a[0], a[1], self.pshift), p)

    def invalidate(self, u, lf, ll):
        gone = [k for k, r in self.m.rec.items() if r[0][0] == u and lf <= r[0][1] <= ll]
        for k in gone:
            del self.m.rec[k]
        return len(gone)

    def live(self):
        return {r[0] for r in self.m.rec.values()}

    def agrees(self, E, eng, pool, small=True):
        u, l = _ua(pool)
        want = {"hit": E.HIT, "miss": E.MISS, "bad entry": E.BAD_ENTRY}
        for fn in ((eng.get, eng.get_small) if small else (eng.get,)):
            out, st = fn(u, l)
            for i, a in enumerate(pool):
                s, page = self.m.get_status(*K.cachemap_args(a[0], a[1], self.pshift))
                assert st[i] == want[s], (fn.__name__, i, a, int(st[i]), s)
                if s == "hit":
                    assert bytes(out[i]) == bytes(page), (fn.__name__, i, a)
        assert eng.entries() == len(self.m.rec)


def _put(eng, model, addrs, pages):
    u, l = _ua(addrs)
    eng.put(u, l, pages)
    model.put(addrs, pages)


def _inv(eng, model, u, lf, ll):
    got = eng.invalidate(u, lf, ll)
    assert got == model.invalidate(u, lf, ll), (u, lf, ll)
    return got


@pytest.mark.parametrize("pshift", [12, 16, 17])
def test_invalidation_matches_the_model(E, gpu, oracle, pshift):
    bs = 1 << pshift
    slots = 4096                                    # keyed up to (4096 + 2) / 64 = 64 addresses, then a scan
    eng = E.Engine(pshift=pshift, accel=12, capacity=2048, table_slots=slots, arena_bytes=512 << 20,
                   max_batch=64, flags=E.FINGERPRINT)
    model = Model(oracle, pshift)
    pool = []
    for nh in (3, 4, 5):
        for gen in (0, 1):
            pages = list(range(40)) + [700, 701, 5000, (1 << 44) - 1]
            pool += [(nh, p | gen << 44) for p in pages]
    for at in range(0, len(pool), 64):
        chunk = pool[at:at + 64]
        _put(eng, model, chunk, _pages(bs, len(chunk), at + pshift))
    model.agrees(E, eng, pool)
    g1 = 1 << 44
    steps = [
        (3, 7, 7),                      # one page (keyed)
        (3, 10, 29),                    # a middle range (keyed)
        (3, 35, (1 << 44) - 1),         # to the end of generation 0 (scan)
        (4, g1 + 5, g1 + 5 + 600),      # generation 1, 601 addresses (scan); generation 0 stays
        (4, 0, 2),                      # keyed, generation 0
        (5, g1, TO_END),                # everything of generation 1 and above (scan)
        (5, 0, 511),                    # 512 addresses (scan)
        (5, 690, 753),                  # keyed at the largest keyed count, 64 addresses
        (3, 0, TO_END),                 # the full interval: all generations of object 3 (scan)
        (6, 0, TO_END),                 # an object with nothing cached
    ]
    for u, lf, ll in steps:
        _inv(eng, model, u, lf, ll)
        model.agrees(E, eng, pool)
        # the same interval again removes nothing
        assert eng.invalidate(u, lf, ll) == 0
    # what was invalidated can be put again
    again = [a for a in pool if a not in model.live()][:64]
    _put(eng, model, again, _pages(bs, len(again), 99))
    model.agrees(E, eng, pool)
    with pytest.raises(RuntimeError):
        eng.invalidate(3, 9, 8)
    eng.close()


@pytest.mark.parametrize("scan", [False, True])
def test_key_edges_remove_only_the_stored_address(E, gpu, oracle, scan):
    fx = K.load()
    pshift = 12
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=64)
    model = Model(oracle, pshift)
    pool = [a for g in fx["groups"].values() for a in g]

    def inv(a):
        return _inv(eng, model, a[0], *((0, TO_END) if scan else (a[1], a[1])))

    for name in ("quad", "pair0", "pair1", "pair2"):
        group = fx["groups"][name]
        for i, a in enumerate(group):
            other = group[(i + 1) % len(group)]
            _put(eng, model, [other], _pages(4096, 1, 7 + i))
            assert inv(a) == 0                              # the key holds `other`: it stays
            model.agrees(E, eng, pool)
            _put(eng, model, [a], _pages(4096, 1, 17 + i))
            assert inv(a) == 1
            model.agrees(E, eng, pool)
    for name in ("key0", "key_ones"):
        a, b = fx["groups"][name][:2]
        _put(eng, model, [b], _pages(4096, 1, 30))
        assert inv(a) == 0
        assert inv(b) == 1                                  # the side slot is emptied
        model.agrees(E, eng, pool)
        _put(eng, model, [a], _pages(4096, 1, 31))          # and takes a record again
        model.agrees(E, eng, pool)
        assert inv(a) == 1
        model.agrees(E, eng, pool)
    assert eng.stats()["entries"] == 0
    eng.close()


def test_host_tier_records_leave_once(E, gpu):
    pshift, bs = 12, 4096
    tier = 256 << 10                                        # ~62 incompressible records per lap
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128, host_tier_bytes=tier)
    pa = np.stack([datagen.make_page("R", bs, 900 + i) for i in range(100)])
    u6, l6 = np.full(100, 6, dtype=np.uint64), np.arange(100, dtype=np.uint64)
    eng.put(u6, l6, pa)
    assert eng.demote(u6[:60], l6[:60]) == 60
    ht0 = eng.host_tier_stats()
    assert ht0["records"] == 60
    assert eng.invalidate(6, 0, 79) == 80                   # 60 from the tier, 20 from the arena
    ht1 = eng.host_tier_stats()
    assert ht1["records"] == 0 and ht1["garbage"] >= ht0["garbage"] + 60 * (bs + 24)
    assert eng.entries() == 20
    # lap the ring over the invalidated records: none of them is retired, entries falls only for the new
    pb = np.stack([datagen.make_page("R", bs, 2000 + i) for i in range(150)])
    u8, l8 = np.full(150, 8, dtype=np.uint64), np.arange(150, dtype=np.uint64)
    eng.put(u8, l8, pb)
    for at in range(0, 150, 50):
        assert eng.demote(u8[at:at + 50], l8[at:at + 50]) == 50
    ht2 = eng.host_tier_stats()
    out, st = eng.get(u8, l8)
    live8 = int((st == E.HIT).sum())
    assert ((st == E.HIT) | (st == E.MISS)).all() and (out[st == E.HIT] == pb[st == E.HIT]).all()
    assert ht2["retired_records"] == 150 - live8
    assert eng.entries() == 20 + live8 and ht2["records"] == live8
    out, st = eng.get(u6, l6)
    assert (st[:80] == E.MISS).all() and (st[80:] == E.HIT).all() and (out[80:] == pa[80:]).all()
    eng.close()


def test_snapshots_and_chains_see_the_invalidation(E, gpu, oracle, tmp_path):
    pshift, bs = 12, 4096
    geo = dict(pshift=pshift, accel=12, capacity=2048, arena_bytes=128 << 20, max_batch=64, flags=E.FINGERPRINT)
    eng = E.Engine(**geo)
    model = Model(oracle, pshift)
    fx = K.load()
    pool = [(9, p) for p in range(120)] + [(10, p) for p in range(40)] + [a for g in fx["groups"].values() for a in g]
    _put(eng, model, pool, _pages(bs, len(pool), 5))
    base = str(tmp_path / "c.snap")
    E.snapshot_finish(E.chain_begin([eng.h], base, False))
    before = model.live()
    s = eng.snapshot_begin(str(tmp_path / "early.snap"))    # begun before the call
    _inv(eng, model, 9, 20, 79)                             # keyed
    _inv(eng, model, 10, 0, TO_END)                         # scan
    E.snapshot_finish(s)
    gone = before - model.live()
    assert len(gone) == 100
    early = {sc.addr_of(r[3]) for r in snapshot.read_snapshot(str(tmp_path / "early.snap"))[2]}
    assert early == before
    eng.save(str(tmp_path / "late.snap"))
    late = {sc.addr_of(r[3]) for r in snapshot.read_snapshot(str(tmp_path / "late.snap"))[2]}
    assert late == model.live()
    E.snapshot_finish(E.chain_begin([eng.h], base, True))
    d = sc.read_delta(base + ".d1")
    assert sorted(d["tombstones"]) == sorted(gone) and d["records"] == []
    e2 = E.Engine(**geo)
    assert E.load_chain([e2.h], base) == (len(model.live()), 1)
    model.agrees(E, e2, pool)
    e2.close()
    eng.close()


def test_verified_gets_miss_invalidated_pages(E, gpu, oracle):
    pshift, bs = 16, 65536
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, arena_bytes=256 << 20, max_batch=64, flags=E.VERIFY)
    model = Model(oracle, pshift)
    pool = [(12, p) for p in range(64)]
    _put(eng, model, pool, _pages(bs, 64, 8))
    _inv(eng, model, 12, 16, 47)
    u, l = _ua(pool)
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st[16:48] == E.MISS).all() and (st[:16] == E.HIT).all() and (st[48:] == E.HIT).all()
    assert eng.verify_stats()["corrupt"] == 0
    _, _, n_bad, checked = eng.verify_store()
    assert n_bad == 0 and checked == 32
    model.agrees(E, eng, pool)
    eng.close()


def test_small_gets_overlap_invalidations_without_torn_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 192, 65536
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=3 << 30, max_batch=256)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 77, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
eng.put(u, l, A)
stop = threading.Event(); bad = []; misses = [0]
def reader():
    while not stop.is_set():
        out, st = eng.get_small(u, l)
        hit = st == E.HIT
        misses[0] += int((st == E.MISS).sum())
        ok = (hit & ((out == A).all(axis=1) | (out == B).all(axis=1))) | (st == E.MISS)
        if not ok.all():
            bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
            return
th = [threading.Thread(target=reader) for _ in range(2)]
[t.start() for t in th]
for rnd in range(40):
    assert eng.invalidate(77, 0 if rnd % 2 else 100, (1 << 64) - 1 if rnd % 2 else 100 + n) > 0
    eng.put(u, l, B if rnd % 2 == 0 else A)
stop.set(); [t.join() for t in th]
assert not bad, bad
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
print("no torn pages", misses[0])
'''
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def test_a_large_invalidation_rebuilds_the_table(E, gpu, oracle):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, table_slots=4096, arena_bytes=64 << 20, max_batch=512,
                   flags=E.FINGERPRINT)
    model = Model(oracle, pshift)
    doomed = [(20, p) for p in range(1200)]
    keep = [(21, p) for p in range(300)]
    _put(eng, model, doomed, _pages(bs, 1200, 2))
    _put(eng, model, keep, _pages(bs, 300, 3))
    assert eng.stats()["tombstones"] == 0
    _inv(eng, model, 20, 0, 1199)
    st = eng.stats()
    assert st["tombstones"] == 0 and st["entries"] == 300          # 1200 > 4096 / 8: rebuilt
    model.agrees(E, eng, keep + doomed[:64])
    u, l = _ua(keep)
    words, ok = eng.read_checkpoints(u, l)
    assert (ok == 1).all(), ok
    recs = eng.read_records(u, l)
    for i, r in enumerate(recs):
        assert words[i, 1:].tolist() == ckpt_words(r[24:], bs)[1:]
    eng.close()


def test_refused_after_a_multi_gpu_call(E, gpu):
    eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64)
    eng.put(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64), _pages(4096, 1, 1))
    assert eng.invalidate(2, 0, TO_END) == 0
    eng.set_stream_order(100, 2)
    with pytest.raises(RuntimeError, match="multi-GPU"):
        eng.invalidate(1, 0, TO_END)
    eng.close()


DROP_IN = textwrap.dedent("""
    import os, shutil, sys, time
    sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
    sys.path.insert(0, sys.argv[1])
    import datagen
    import edge_fuse_b200 as E
    d, phase = sys.argv[2], sys.argv[3]
    P = 4096
    old = [datagen.make_page("RTZMPAXS"[i % 8], P, 100 + i) for i in range(32)]
    new = [datagen.make_page("RTZMPAXS"[i % 8], P, 500 + i) for i in range(20)]
    TO, FROM = 50, 51

    def misses(cm):
        gone = sum(cm.get(i * P, TO, 0) is None for i in range(32))
        gone += sum(cm.get(i * P, FROM, 0) is None for i in range(20))
        return gone, cm.read_range(TO, 0, 0, 20 * P) is None, cm.read_range(FROM, 0, 0, 20 * P) is None

    if phase in ("write", "crash"):
        cm = E.Cachemap(d, 4096, 12, 12)
        for i in range(32):
            cm.put(i * P, TO, 0, old[i])                  # the file the rename replaces
        for i in range(20):
            cm.put(i * P, FROM, 0, new[i])                # f.tmp, written and read back
        assert cm.read_range(TO, 0, 0, 32 * P) is not None and cm.read_range(FROM, 0, 0, 20 * P) is not None
        if phase == "crash":
            time.sleep(2.5)                               # a base is written
        # rename(FROM, TO): the server copies FROM to TO and deletes FROM; the cache drops both names
        removed = cm.invalidate(TO, 0, 0, E.Cachemap.TO_END) + cm.invalidate(FROM, 0, 0, E.Cachemap.TO_END)
        print("removed", removed, "misses", *misses(cm), flush=True)
        if phase == "crash":
            time.sleep(2.5)                               # a delta tick holds the removal
            shutil.copytree(d, d + ".copy")
            print("files", " ".join(sorted(os.listdir(d + ".copy"))), flush=True)
            os._exit(0)
        cm.free()
    else:
        cm = E.Cachemap(d, 4096, 12, 12)
        print("misses", *misses(cm), flush=True)
        cm.free()
""")


@pytest.mark.parametrize("crash", [False, True])
def test_drop_in_rename_over_two_engines(E, gpu, tmp_path, crash):
    script = tmp_path / "drive.py"
    script.write_text(DROP_IN)
    env = dict(os.environ, CMB200_DEVICES="0,0", CMB200_PERSIST="1", CMB200_ARENA_MB="256")
    for k in ("CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        env.pop(k, None)
    if crash:
        env.update(CMB200_CHECKPOINT_SEC="1", CMB200_CHECKPOINT_DELTAS="4")
    d = tmp_path / "cache"
    d.mkdir()
    w = subprocess.run([sys.executable, str(script), ROOT, str(d), "crash" if crash else "write"],
                       capture_output=True, text=True, timeout=300, env=env)
    assert w.returncode == 0 and "removed 52 misses 52 True True" in w.stdout, w.stdout + w.stderr[-3000:]
    if crash:
        assert "cachemap_b200.snap.d" in w.stdout, w.stdout
        d = tmp_path / "cache.copy"
    r = subprocess.run([sys.executable, str(script), ROOT, str(d), "read"], capture_output=True, text=True,
                       timeout=300, env=env)
    assert r.returncode == 0 and "misses 52 True True" in r.stdout, r.stdout + r.stderr[-3000:]
    shutil.rmtree(tmp_path / "cache", ignore_errors=True)
