"""GPU tests of cmb200_rename / cmb200_rename_set and cachemap_rename: every live record of {u_from, l},
l in an interval, moves to {u_to, l} byte for byte as a put of the same page there would store it, with
its ts and fingerprint, and with parse checkpoints rebuilt; the old address is served by no get.
Checked against the reference's record bytes, a store model, both selection paths, shared and sentinel
keys, the host tier, eviction by access, drops, compaction between slices, snapshots and chains,
concurrent small gets, the multi-GPU refusal, and the drop-in over two engines."""
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


def _pages(bs, n, seed, kinds="RTZMPAXS"):
    return np.stack([datagen.make_page(kinds[(seed + i) % len(kinds)], bs, seed * 131 + i) for i in range(n)])


class Model:
    """oracle.StoreModel with rename: a record of {u_from, l} in the interval becomes a put of its page at
    {u_to, l} (same block), and its old key is removed.  Addresses are (u, l) pairs."""

    def __init__(self, oracle, pshift, accel=12):
        self.O, self.pshift = oracle, pshift
        self.m = oracle.StoreModel(pshift, accel)

    def put(self, addrs, pages):
        for a, p in zip(addrs, pages):
            self.m.put(*K.cachemap_args(a[0], a[1], self.pshift), p)

    def rename(self, uf, ut, lf, ll, dropped=()):
        moving = sorted((r for r in self.m.rec.values() if r[0][0] == uf and lf <= r[0][1] <= ll),
                        key=lambda r: r[0][1])
        for r in moving:
            del self.m.rec[self.O.addr_key(*r[0])]
        for r in moving:
            a = (ut, r[0][1])
            if a not in dropped:
                self.m.rec[self.O.addr_key(*a)] = (a, r[1], r[2])
        return len(moving)

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
        recs = eng.read_records(u, l)
        for i, a in enumerate(pool):
            if a in self.live():
                assert recs[i] == self.m.record_bytes(*a), a
        assert eng.entries() == len(self.m.rec)


def _ts_by_addr(eng, path):
    eng.save(path)
    return {sc.addr_of(r[3]): (r[0], r[1], r[2]) for r in snapshot.read_snapshot(path)[2]}


@pytest.mark.parametrize("pshift", [12, 16, 17, 20])
def test_moved_records_equal_a_put_at_the_new_name(E, gpu, oracle, tmp_path, pshift):
    bs = 1 << pshift
    n = 24 if pshift < 20 else 8
    flags = E.VERIFY | E.FINGERPRINT
    geo = dict(pshift=pshift, accel=12, capacity=1024, arena_bytes=max(256 << 20, 4 * n * (bs + 2048)),
               max_batch=64, flags=flags)
    moved_eng, put_eng = E.Engine(**geo), E.Engine(**geo)
    # R pages stay raw above 128 KiB; the rest compress
    pages = _pages(bs, n, pshift, kinds="RTZMPAXS")
    uf, ut = 41, 42
    ls = np.arange(n, dtype=np.uint64) + 3
    ts = np.arange(n, dtype=np.uint64) * 1000 + 77
    moved_eng.put(np.full(n, uf, dtype=np.uint64), ls, pages, ts=ts)
    put_eng.put(np.full(n, ut, dtype=np.uint64), ls, pages, ts=ts)
    assert moved_eng.rename(uf, ut, 0, TO_END) == (n, 0)
    uto, ufr = np.full(n, ut, dtype=np.uint64), np.full(n, uf, dtype=np.uint64)
    got, want = moved_eng.read_records(uto, ls), put_eng.read_records(uto, ls)
    model = Model(oracle, pshift)
    model.put([(ut, int(x)) for x in ls], pages)
    for i in range(n):
        assert got[i] == want[i] == model.m.record_bytes(ut, int(ls[i])), i
    assert all(r is None for r in moved_eng.read_records(ufr, ls))
    fa, oka = moved_eng.read_fingerprints(uto, ls)
    fb, okb = put_eng.read_fingerprints(uto, ls)
    assert (oka == 1).all() and (okb == 1).all() and (fa == fb).all()
    if pshift <= 17:
        wa, ca = moved_eng.read_checkpoints(uto, ls)
        wb, cb = put_eng.read_checkpoints(uto, ls)
        assert (ca == cb).all() and (wa[:, 1:] == wb[:, 1:]).all()
        for i, r in enumerate(got):
            if ca[i] == 1:
                assert wa[i, 1:].tolist() == ckpt_words(r[24:], bs)[1:]
    # ts and fingerprints as a snapshot sees them
    sa = _ts_by_addr(moved_eng, str(tmp_path / "a.snap"))
    sb = _ts_by_addr(put_eng, str(tmp_path / "b.snap"))
    assert sa == sb
    # gets: the new name hits with the page, verified; the old one misses
    for fn in (moved_eng.get, moved_eng.get_small) if pshift <= 17 else (moved_eng.get,):
        out, st = fn(uto, ls)
        assert (st == E.HIT).all() and (out == pages).all(), fn.__name__
        _, st = fn(ufr, ls)
        assert (st == E.MISS).all(), fn.__name__
    vs = moved_eng.verify_stats()
    assert vs["unverified"] == 0 and vs["corrupt"] == 0 and vs["verified"] >= n
    moved_eng.close()
    put_eng.close()


@pytest.mark.parametrize("pshift", [12, 17])
def test_keyed_and_scan_selection_leave_the_same_store(E, gpu, oracle, pshift):
    bs = 1 << pshift
    geo = dict(pshift=pshift, accel=12, capacity=2048, table_slots=4096, arena_bytes=512 << 20, max_batch=64,
               flags=E.FINGERPRINT)
    pool = []
    for nh in (3, 4):
        for gen in (0, 1):
            pool += [(nh, p | gen << 44) for p in list(range(40)) + [700, 5000, (1 << 44) - 1]]
    pages = _pages(bs, len(pool), pshift)
    engs, models = [E.Engine(**geo), E.Engine(**geo)], [Model(oracle, pshift), Model(oracle, pshift)]
    for eng, model in zip(engs, models):
        for at in range(0, len(pool), 64):
            eng.put(*_ua(pool[at:at + 64]), pages[at:at + 64])
            model.put(pool[at:at + 64], pages[at:at + 64])
    check = pool + [(7, a[1]) for a in pool] + [(8, a[1]) for a in pool]
    # keyed: intervals of at most (4096 + 2) / 64 = 64 addresses, one per call; scan: the same pages in
    # longer intervals
    keyed = [(3, 7, 0, 39), (3, 7, 700, 700), (4, 8, 1 << 44, (1 << 44) + 63), (3, 7, (1 << 44) - 1, (1 << 44) - 1)]
    scan = [(3, 7, 0, 700), (4, 8, 1 << 44, (1 << 44) + 650), (3, 7, (1 << 44) - 65, (1 << 44) - 1)]
    for eng, model, steps in ((engs[0], models[0], keyed), (engs[1], models[1], scan)):
        for uf, ut, lf, ll in steps:
            got = eng.rename(uf, ut, lf, ll)
            assert got == (model.rename(uf, ut, lf, ll), 0), (uf, ut, lf, ll)
            model.agrees(E, eng, check, small=pshift <= 17)
    assert models[0].live() == models[1].live()
    u, l = _ua(check)
    assert engs[0].read_records(u, l) == engs[1].read_records(u, l)
    with pytest.raises(RuntimeError):
        engs[0].rename(3, 7, 9, 8)
    assert engs[0].rename(4, 4, 0, TO_END) == (0, 0)
    for e in engs:
        e.close()


def test_key_edges_replace_as_a_put_and_leave_other_addresses(E, gpu, oracle):
    fx = K.load()
    pshift = 12
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, table_slots=4096, arena_bytes=64 << 20, max_batch=64)
    model = Model(oracle, pshift)
    pool = [a for g in fx["groups"].values() for a in g]
    uf = 0x5151
    pool += [(uf, a[1]) for a in pool]
    seed = 0
    for name in ("quad", "pair0", "pair1", "pair2", "key0", "key_ones"):
        a, b = fx["groups"][name][:2]
        seed += 1
        # the new address's key holds another address: the moved record replaces it, as a put would
        eng.put(*_ua([b]), _pages(4096, 1, seed))
        model.put([b], _pages(4096, 1, seed))
        eng.put(*_ua([(uf, a[1])]), _pages(4096, 1, seed + 50))
        model.put([(uf, a[1])], _pages(4096, 1, seed + 50))
        for scan in (False, True):
            lf, ll = (0, TO_END) if scan else (a[1], a[1])
            got = eng.rename(uf, a[0], lf, ll)
            assert got == (model.rename(uf, a[0], lf, ll), 0), (name, scan)
            model.agrees(E, eng, pool)
        # an old address whose key holds another address is not touched
        eng.put(*_ua([b]), _pages(4096, 1, seed + 100))
        model.put([b], _pages(4096, 1, seed + 100))
        for scan in (False, True):
            lf, ll = (0, TO_END) if scan else (a[1], a[1])
            assert eng.rename(a[0], uf, lf, ll) == (model.rename(a[0], uf, lf, ll), 0), (name, scan)
            assert b in model.live()
            model.agrees(E, eng, pool)
    eng.close()


def test_host_tier_records_move_into_the_arena(E, gpu, oracle):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128,
                   host_tier_bytes=1 << 20)
    model = Model(oracle, pshift)
    pool = [(6, p) for p in range(100)]
    pages = _pages(bs, 100, 3, kinds="R")
    eng.put(*_ua(pool), pages)
    model.put(pool, pages)
    u, l = _ua(pool)
    assert eng.demote(u[:60], l[:60]) == 60
    ht0 = eng.host_tier_stats()
    assert ht0["records"] == 60
    assert eng.rename(6, 9, 0, TO_END) == (100, 0)
    model.rename(6, 9, 0, TO_END)
    ht1 = eng.host_tier_stats()
    assert ht1["records"] == 0 and ht1["garbage"] >= ht0["garbage"] + 60 * (bs + 24)
    check = pool + [(9, p) for p in range(100)]
    model.agrees(E, eng, check)
    # nothing of the new name is answered from the tier
    assert eng.host_tier_stats()["hits"] == ht1["hits"]
    eng.close()


def test_access_stamps_survive_the_move(E, gpu, tmp_path):
    pshift, bs = 12, 4096
    eng = E.Engine(pshift=pshift, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, flags=E.TOUCH)
    n = 32
    pages = _pages(bs, n, 5)
    u, l = np.full(n, 11, dtype=np.uint64), np.arange(n, dtype=np.uint64)
    eng.put(u, l, pages, ts=np.arange(n, dtype=np.uint64) + 5)
    eng.get_small(u[:8], l[:8])                     # raises ts of the first eight to the clock
    before = _ts_by_addr(eng, str(tmp_path / "a.snap"))
    assert eng.rename(11, 12, 0, TO_END) == (n, 0)
    after = _ts_by_addr(eng, str(tmp_path / "b.snap"))
    assert {(12, a[1]): v for a, v in before.items()} == after
    assert all(after[(12, i)][0] > 10 ** 15 for i in range(8))
    eng.close()


def test_a_full_destination_drops_and_nothing_stale_is_served(E, gpu, oracle):
    pshift, bs = 12, 4096
    big = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=64, device=0)
    small = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=96 << 10, max_batch=64, device=0)
    engs = [big, small]
    n = 200
    pages = _pages(bs, n, 9, kinds="R")             # incompressible: ~4 KiB records
    uf, ut = 21, 22
    fr = [(uf, p) for p in range(n)]
    # the old pages of the new name, on the small engine, fill most of its arena with live records
    old = [(ut, p) for p in range(n) if E.owner(oracle.addr_key(ut, p), 2) == 1][:20]
    small.put(*_ua(old), _pages(bs, len(old), 1, kinds="R"))
    small.unset(*_ua(old))                          # the caller invalidates the new name first
    filler = [(99, p) for p in range(1000) if E.owner(oracle.addr_key(99, p), 2) == 1][:2]
    small.put(*_ua(filler), _pages(bs, len(filler), 2, kinds="R"))
    big.put(*_ua(fr), pages)                        # the move reads every engine, whichever owns the key
    assert big.stats()["dropped_puts"] == 0
    dropped_before = small.stats()["dropped_puts"]
    moved, dropped = E.rename_set([big.h, small.h], uf, ut, 0, TO_END)
    assert moved + dropped == n and dropped > 0 and moved > 0
    assert small.stats()["dropped_puts"] - dropped_before == dropped
    hits = 0
    for e in engs:
        out, st = e.get(*_ua(fr))
        assert (st == E.MISS).all()
        to = [(ut, p) for p in range(n)]
        out, st = e.get(*_ua(to))
        assert ((st == E.HIT) | (st == E.MISS)).all()
        for i in np.nonzero(st == E.HIT)[0]:
            assert (out[i] == pages[i]).all()
        hits += int((st == E.HIT).sum())
    assert hits == moved
    for e in engs:
        e.close()


def test_compaction_between_slices_and_a_move_of_many_slices(E, gpu, oracle):
    pshift, bs = 12, 4096
    n = 600                                          # > max_batch: many slices
    # room for the live records and about a third more: the move must compact to fit
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=int(n * (bs + 32) * 1.35), max_batch=32,
                   flags=E.FINGERPRINT)
    model = Model(oracle, pshift)
    pool = [(31, p) for p in range(n)]
    pages = _pages(bs, n, 4, kinds="R")
    eng.put(*_ua(pool), pages)
    model.put(pool, pages)
    st0 = eng.stats()
    assert st0["dropped_puts"] == 0
    moved = eng.rename(31, 32, 0, TO_END)
    assert moved == (model.rename(31, 32, 0, TO_END), 0)
    st = eng.stats()
    # the arena holds the records and a third more: without a compaction most of the move would drop
    assert st["dropped_puts"] == 0 and st["arena_used"] < st0["arena_used"] + n * (bs + 32) // 2, st
    model.agrees(E, eng, pool + [(32, p) for p in range(n)])
    eng.close()


def test_snapshots_and_chains_after_the_move(E, gpu, oracle, tmp_path):
    pshift, bs = 12, 4096
    geo = dict(pshift=pshift, accel=12, capacity=2048, arena_bytes=128 << 20, max_batch=64, flags=E.FINGERPRINT)
    eng = E.Engine(**geo)
    model = Model(oracle, pshift)
    pool = [(13, p) for p in range(90)] + [(14, p) for p in range(30)]
    pages = _pages(bs, len(pool), 6)
    eng.put(*_ua(pool), pages)
    model.put(pool, pages)
    base = str(tmp_path / "c.snap")
    E.snapshot_finish(E.chain_begin([eng.h], base, False))
    before = model.live()
    assert eng.rename(13, 15, 10, 69) == (model.rename(13, 15, 10, 69), 0)
    check = pool + [(15, p) for p in range(90)]
    E.snapshot_finish(E.chain_begin([eng.h], base, True))
    d = sc.read_delta(base + ".d1")
    assert sorted(d["tombstones"]) == sorted(before - model.live())
    assert sorted(sc.addr_of(r[3]) for r in d["records"]) == sorted(model.live() - before)
    eng.save(str(tmp_path / "full.snap"))
    for load in ("snap", "chain"):
        e2 = E.Engine(**geo)
        if load == "snap":
            e2.load(str(tmp_path / "full.snap"))
        else:
            assert E.load_chain([e2.h], base) == (len(model.live()), 1)
        model.agrees(E, e2, check)
        u, l = _ua(check)
        assert e2.read_records(u, l) == eng.read_records(u, l)
        e2.close()
    eng.close()


def test_small_gets_overlap_renames_without_torn_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 192, 65536
# an arena of 40 MiB: the moves fill it with the garbage they leave, so renames compact (and close
# get_gate) while the readers run
arena = 40 << 20
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=arena, max_batch=64)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
l = np.arange(n, dtype=np.uint64)
names = (np.full(n, 77, dtype=np.uint64), np.full(n, 78, dtype=np.uint64))
eng.put(names[0], l, A)
live = eng.stats()["arena_used"]
assert 2 * live < arena and 40 * live > 2 * arena, live
stop = threading.Event(); bad = []; seen = [0, 0]
def reader(k):
    while not stop.is_set():
        for u in names:
            out, st = eng.get_small(u, l)
            hit = st == E.HIT
            seen[0] += int(hit.sum()); seen[1] += int((st == E.MISS).sum())
            ok = (hit & (out == A).all(axis=1)) | (st == E.MISS)
            if not ok.all():
                bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
                return
th = [threading.Thread(target=reader, args=(k,)) for k in range(2)]
[t.start() for t in th]
for rnd in range(40):
    f, t = (77, 78) if rnd % 2 == 0 else (78, 77)
    assert eng.rename(f, t, 0, (1 << 64) - 1 if rnd % 4 < 2 else n - 1) == (n, 0)
stop.set(); [t.join() for t in th]
assert not bad, bad
# 40 moves allocate 20 times the arena: without compactions inside them the moves would drop pages
assert eng.stats()["dropped_puts"] == 0, eng.stats()
out, st = eng.get_small(names[0], l)
assert (st == E.HIT).all() and (out == A).all()
print("no torn pages", *seen)
'''
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def test_refused_after_a_multi_gpu_call(E, gpu):
    eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64)
    eng.put(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64), _pages(4096, 1, 1))
    assert eng.rename(2, 3, 0, TO_END) == (0, 0)
    eng.set_stream_order(100, 2)
    with pytest.raises(RuntimeError, match="multi-GPU"):
        eng.rename(1, 3, 0, TO_END)
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

    def state(cm):
        right = sum(cm.get(i * P, TO, 0) is not None and bytes(cm.get(i * P, TO, 0)) == bytes(new[i])
                    for i in range(20))
        gone = sum(cm.get(i * P, TO, 0) is None for i in range(20, 32))
        gone += sum(cm.get(i * P, FROM, 0) is None for i in range(20))
        whole = cm.read_range(TO, 0, 0, 20 * P)
        return right, gone, whole is not None and bytes(whole) == b"".join(bytes(p) for p in new)

    if phase in ("write", "crash"):
        cm = E.Cachemap(d, 4096, 12, 12)
        for i in range(32):
            cm.put(i * P, TO, 0, old[i])                  # the file the rename replaces, larger
        for i in range(20):
            cm.put(i * P, FROM, 0, new[i])                # f.tmp, written
        if phase == "crash":
            time.sleep(2.5)                               # a base is written
        moved = cm.rename(FROM, TO, 0)                    # rename(FROM, TO)
        print("moved", moved, "state", *state(cm), flush=True)
        if phase == "crash":
            time.sleep(2.5)                               # a delta tick holds the move
            shutil.copytree(d, d + ".copy")
            print("files", " ".join(sorted(os.listdir(d + ".copy"))), flush=True)
            os._exit(0)
        cm.free()
    else:
        cm = E.Cachemap(d, 4096, 12, 12)
        print("state", *state(cm), flush=True)
        cm.free()
""")


@pytest.mark.parametrize("devices,crash", [("0,0", False), ("0,0", True), ("all", False)])
def test_drop_in_rename_over_several_engines(E, gpu, tmp_path, devices, crash):
    if devices == "all" and gpu < 2:
        pytest.skip("one GPU: CMB200_DEVICES=all is one engine, covered by 0,0")
    script = tmp_path / "drive.py"
    script.write_text(DROP_IN)
    env = dict(os.environ, CMB200_DEVICES=devices, CMB200_PERSIST="1", CMB200_ARENA_MB="256")
    for k in ("CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        env.pop(k, None)
    if crash:
        env.update(CMB200_CHECKPOINT_SEC="1", CMB200_CHECKPOINT_DELTAS="4")
    d = tmp_path / "cache"
    d.mkdir()
    w = subprocess.run([sys.executable, str(script), ROOT, str(d), "crash" if crash else "write"],
                       capture_output=True, text=True, timeout=300, env=env)
    assert w.returncode == 0 and "moved 20 state 20 32 True" in w.stdout, w.stdout + w.stderr[-3000:]
    if crash:
        assert "cachemap_b200.snap.d" in w.stdout, w.stdout
        d = tmp_path / "cache.copy"
    r = subprocess.run([sys.executable, str(script), ROOT, str(d), "read"], capture_output=True, text=True,
                       timeout=300, env=env)
    assert r.returncode == 0 and "state 20 32 True" in r.stdout, r.stdout + r.stderr[-3000:]
    shutil.rmtree(tmp_path / "cache", ignore_errors=True)


# ---- the store machine of tests/store_machine.py with renames ----------------------------------------
# The seeded logs of store_machine.gen_ops with rename(u_from, u_to, l_first, l_last) steps inserted
# from a generator of their own (the logs' own seeds and steps are unchanged), run through the GPU
# driver of tests/test_gpu_store_machine.py and checked against the model after every step.
import dataclasses  # noqa: E402

import store_machine as SM  # noqa: E402
import test_gpu_store_machine as GSM  # noqa: E402


class RenameModel(SM.Model):
    def rename(self, uf, ut, lf, ll, dropped_ls) -> int:
        """cmb200_rename: each record of {uf, l} in the interval leaves its key and is stored at {ut, l}
        as a put of its page there would store it, with its ts and fingerprint; the rows the engine
        dropped (`dropped_ls`, by l) store nothing and count as dropped puts."""
        cfg = self.cfg
        moving = sorted((r for r in self.rec.values() if r.addr[0] == uf and lf <= r.addr[1] <= ll),
                        key=lambda r: r.addr[1])
        if not moving:
            return 0
        total = sum(r.need for r in moving)
        one_slice = len(moving) <= cfg.max_batch and total <= min(cfg.max_batch, 4096) * cfg.bsize
        for r in moving:
            self._remove(self.key(r.addr))
        # the engine checks for a table rebuild after every slice: keep only the upper bound
        self.tomb_lo = 0
        uncertain = False
        # the bump pointer is predicted for a one-slice move of an exactly tracked arena; otherwise the
        # driver reads it back from the engine (head_known False)
        self.head_known = cfg.exact_head and not self.saturated and one_slice
        if self.head_known:
            # one slice: the sources are garbage now; one compaction if garbage covers the shortfall
            short = self.head + total - self.arena_size
            if short > 0 and self.head - self.arena_alloc() >= short:
                self.compact()
        elif self.head + total > self.arena_size:
            uncertain = True                         # a compaction or drops in some slice
        for r in moving:
            a = (ut, r.addr[1])
            self.head += r.need
            if r.addr[1] in dropped_ls:
                self.ctr.dropped += 1
                continue
            self._install(dataclasses.replace(r, addr=a, host_pos=None))
        if dropped_ls or uncertain:
            self.saturated = True
        return len(moving)


def gen_rename_ops(cfg, seed):
    R = SM._Rng(seed * 1009 + 17)
    out = []
    for op in SM.gen_ops(cfg, seed):
        out.append(op)
        if not R.chance(0.12):
            continue
        i = R.below(len(cfg.us))
        uf, ut = cfg.us[i], cfg.us[(i + 1 + R.below(len(cfg.us) - 1)) % len(cfg.us)]
        kind = R.below(3)
        if kind == 0:                                # keyed at every geometry (<= 16 addresses)
            lf = R.below(cfg.nl)
            ll = lf + R.below(16)
        elif kind == 1:                              # scan at every geometry (>= 65 addresses)
            lf = R.below(cfg.nl // 2)
            ll = lf + 64 + R.below(cfg.nl)
        else:
            lf, ll = 0, TO_END
        out.append(("rename", uf, ut, lf, ll))
    return out


class RenameMachine(GSM.Machine):
    def __init__(self, E, oracle, cfg, seed, tmp_path):
        super().__init__(E, oracle, cfg, seed, tmp_path)
        self.m = RenameModel(cfg, oracle)
        self.renames = [0, 0, 0]                     # calls, records moved, records dropped

    def run(self):
        for step, op in enumerate(gen_rename_ops(self.cfg, self.seed)):
            self.log.append(f"{step:4d} {op if op[0] == 'rename' else SM.describe(op)}")
            try:
                getattr(self, "op_" + op[0])(op, step)
                self.check(op[0])
            except AssertionError as e:
                raise AssertionError(f"config {self.cfg.name} seed {self.seed} step {step} ({op[0]}): {e}\n"
                                     "op log (replay: gen_rename_ops(CONFIGS[config], seed)):\n"
                                     + "\n".join(self.log[-60:])) from None
        self.eng.close()
        return self.renames

    def op_rename(self, op, step):
        _, uf, ut, lf, ll = op
        m, eng = self.m, self.eng
        moving = [r.addr[1] for r in m.rec.values() if r.addr[0] == uf and lf <= r.addr[1] <= ll]
        moved, dropped = eng.rename(uf, ut, lf, ll)
        assert moved + dropped == len(moving), f"rename moved {moved} + dropped {dropped}, model {len(moving)}"
        dropped_ls = set()
        if dropped:
            # a dropped row stores nothing: the new address keeps whatever record its key held, as after
            # a dropped put, so a drop shows as a new address that does not hold the moved record
            by_l = {r.addr[1]: r for r in m.rec.values() if r.addr[0] == uf and lf <= r.addr[1] <= ll}
            recs = eng.read_records(np.full(len(moving), ut, dtype=np.uint64), np.array(moving, dtype=np.uint64))
            dropped_ls = {l for l, x in zip(moving, recs)
                          if x != self.O.record_prefix(ut, l, by_l[l].clen) + by_l[l].block}
            assert len(dropped_ls) == dropped, f"{dropped} dropped, {len(dropped_ls)} new addresses lack the moved record"
        if m.rename(uf, ut, lf, ll, dropped_ls) and self.cfg.exact_head and not m.head_known:
            m.head = eng.stats()["arena_used"]       # a slice compacted or dropped where the model cannot see
        self.renames[0] += 1
        self.renames[1] += moved
        self.renames[2] += dropped


@pytest.mark.parametrize("name,seed", [(n, s) for n in sorted(SM.CONFIGS) for s in SM.CONFIGS[n].seeds])
def test_store_machine_with_renames(E, gpu, oracle, tmp_path, monkeypatch, name, seed):
    cfg = SM.CONFIGS[name]
    for k in ("CMB200_SEG_KB", "CMB200_CKPT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in cfg.env:
        monkeypatch.setenv(k, v)
    calls, moved, _dropped = RenameMachine(E, oracle, cfg, seed, tmp_path).run()
    assert calls >= 3 and moved > 0, (calls, moved)
