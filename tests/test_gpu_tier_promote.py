"""GPU tests of promotion from the host tier back to the HBM arena (cmb200_promote_batch), of the log of
tier hits that tells the engine which tier keys are hot (cmb200_host_tier_hot), and of the drop-in's
CMB200_TIER_PROMOTE policy built on the two."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import datagen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need(rec_len):
    return (rec_len + 15) & ~15


def _keys(tag, n, start=0):
    return np.full(n, tag, dtype=np.uint64), np.arange(start, start + n, dtype=np.uint64)


@pytest.mark.parametrize("pshift", [12, 16])
@pytest.mark.parametrize("accel", [12, 0])
def test_promoted_records_are_the_references_bytes(E, gpu, oracle, pshift, accel):
    bs, n, kinds = 1 << pshift, 70, "RTZMPAX"
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], bs, 300 + i) for i in range(n)])
    eng = E.Engine(pshift=pshift, accel=accel, capacity=4096, arena_bytes=64 << 20, max_batch=64,
                   host_tier_bytes=64 << 20)
    u, l = _keys(41, n)
    eng.put(u, l, pages)
    assert eng.demote(u, l) == n
    au, al = _keys(43, 6)                                          # keys that stay in the arena
    apages = pages[:6].copy()
    eng.put(au, al, apages)
    recs = eng.read_records(u, l)
    p = 35                                                         # promote keys 0..34
    su = np.concatenate([u[:20], au, u[:5], [np.uint64(42)], u[20:p], u[30:p]])
    sl = np.concatenate([l[:20], al, l[:5], [np.uint64(0)], l[20:p], l[30:p]])
    s0, h0 = eng.stats(), eng.host_tier_stats()
    assert eng.promote(su, sl) == p
    assert eng.promote(su, sl) == 0                                # all in the arena now
    s1, h1 = eng.stats(), eng.host_tier_stats()
    moved = sum(_need(len(r)) for r in recs[:p])
    assert s1["entries"] == s0["entries"] == n + 6
    assert s1["arena_used"] - s0["arena_used"] == moved
    assert h1["records"] == h0["records"] - p and h1["garbage"] - h0["garbage"] == moved
    assert h1["promoted_records"] == p and h1["promoted_bytes"] == sum(len(r) for r in recs[:p])
    assert h1["demoted_records"] == h0["demoted_records"] and s1["dropped_puts"] == 0
    assert eng.read_records(u, l) == recs
    for i in range(n):
        blk = pages[i].tobytes() if accel == 0 else oracle.lz4_encode(pages[i], accel)
        assert recs[i] == oracle.record_prefix(int(u[i]), int(l[i]), 0 if accel == 0 else len(blk)) + blk, i
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
        out, st = fn(au, al)
        assert (st == E.HIT).all() and (out == apages).all()
    hits = eng.host_tier_stats()["hits"]
    assert hits == 2 * (n - p)                                     # the promoted keys were read from the arena
    for fn in (eng.get, eng.get_small):
        fn(u[:p], l[:p])
    assert eng.host_tier_stats()["hits"] == hits
    eng.close()


def test_promotion_at_128k_pages_through_the_pair_kernel(E, gpu):
    bs, n = 1 << 17, 6
    pages = np.stack([datagen.make_page("TZM"[i % 3], bs, 40 + i) for i in range(n)])
    eng = E.Engine(pshift=17, accel=12, capacity=1024, arena_bytes=64 << 20, max_batch=64, host_tier_bytes=16 << 20)
    u, l = _keys(17, n)
    eng.put(u, l, pages)
    recs = eng.read_records(u, l)
    assert eng.demote(u, l) == n
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all() and eng.host_tier_stats()["hits"] == n
    assert eng.promote(u[:4], l[:4]) == 4
    ht = eng.host_tier_stats()
    assert ht["records"] == n - 4 and ht["promoted_bytes"] == sum(len(r) for r in recs[:4])
    assert eng.read_records(u, l) == recs
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    assert eng.host_tier_stats()["hits"] == n + (n - 4)
    eng.close()


def test_promotion_uses_free_arena_bytes_only(E, gpu):
    bs, n = 4096, 300
    eng = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=1 << 20, max_batch=128, host_tier_bytes=4 << 20)
    pages = np.stack([datagen.make_page("R", bs, 2000 + i) for i in range(n)])
    u, l = _keys(12, n)
    for base in range(0, n, 100):                                  # the arena holds ~250 of these
        eng.put(u[base:base + 100], l[base:base + 100], pages[base:base + 100])
        assert eng.demote(u[base:base + 100], l[base:base + 100]) == 100
        eng.compact()
    recs = eng.read_records(u, l)
    need = {_need(len(r)) for r in recs}
    assert len(need) == 1
    s0 = eng.stats()
    k = (s0["arena_bytes"] - s0["arena_used"]) // need.pop()
    assert 0 < k < n
    assert eng.promote(u, l) == k
    s1, ht = eng.stats(), eng.host_tier_stats()
    assert s1["dropped_puts"] == 0 and s1["entries"] == n and ht["records"] == n - k and ht["retired_records"] == 0
    h0 = ht["hits"]
    out, st = eng.get_small(u[:k], l[:k])                          # array order: the first k moved
    assert (st == E.HIT).all() and (out == pages[:k]).all() and eng.host_tier_stats()["hits"] == h0
    out, st = eng.get_small(u[k:], l[k:])
    assert (st == E.HIT).all() and (out == pages[k:]).all() and eng.host_tier_stats()["hits"] == h0 + n - k
    assert eng.promote(u, l) == 0                                  # still no room
    eng.close()


def test_overwrite_unset_wrap_and_compaction_after_promotion(E, gpu):
    bs, n = 4096, 60
    tier = 256 << 10                                               # ~62 incompressible records per lap
    eng = E.Engine(pshift=12, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128, host_tier_bytes=tier)
    pages = np.stack([datagen.make_page("R", bs, 3000 + i) for i in range(n)])
    newer = np.stack([datagen.make_page("T", bs, 3100 + i) for i in range(5)])
    u, l = _keys(14, n)
    eng.put(u, l, pages)
    assert eng.demote(u, l) == n
    assert eng.promote(u[:20], l[:20]) == 20
    eng.put(u[:5], l[:5], newer)                                   # overwrite promoted keys
    eng.unset(u[5:10], l[5:10])                                    # unset promoted keys
    want = pages.copy()
    want[:5] = newer
    live = np.r_[0:5, 10:n]
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st[5:10] == E.MISS).all() and (st[live] == E.HIT).all() and (out[live] == want[live]).all()
    assert eng.entries() == n - 5
    # lap the tier: the keys still in it are retired, the promoted ones are not
    m = 80
    xu, xl = _keys(15, m)
    extra = np.stack([datagen.make_page("R", bs, 3200 + i) for i in range(m)])
    eng.put(xu, xl, extra)
    for base in range(0, m, 20):
        assert eng.demote(xu[base:base + 20], xl[base:base + 20]) == 20
    keep = np.r_[0:5, 10:20]
    for fn in (eng.get, eng.get_small):
        out, st = fn(u[keep], l[keep])
        assert (st == E.HIT).all() and (out == want[keep]).all()
        _, st_t = fn(u[20:], l[20:])
        _, st_x = fn(xu, xl)
        assert ((st_t == E.HIT) | (st_t == E.MISS)).all() and ((st_x == E.HIT) | (st_x == E.MISS)).all()
    gone = int((st_t == E.MISS).sum() + (st_x == E.MISS).sum())
    ht = eng.host_tier_stats()
    assert gone > 0 and ht["retired_records"] == gone
    assert eng.entries() == len(keep) + (n - 20 - int((st_t == E.MISS).sum())) + (m - int((st_x == E.MISS).sum()))
    eng.compact()
    out, st = eng.get_small(u[keep], l[keep])
    assert (st == E.HIT).all() and (out == want[keep]).all()
    hit_x = st_x == E.HIT
    out, st = eng.get(xu, xl)
    assert (st[hit_x] == E.HIT).all() and (out[hit_x] == extra[hit_x]).all()
    eng.close()


def test_hot_log_names_the_tier_keys_that_gets_read(E, gpu):
    bs, n = 4096, 40
    eng = E.Engine(pshift=12, accel=12, capacity=8192, arena_bytes=64 << 20, max_batch=4096, host_tier_bytes=16 << 20)
    pages = np.stack([datagen.make_page("TZ"[i & 1], bs, 4000 + i) for i in range(n)])
    u, l = _keys(21, n)
    eng.put(u, l, pages)
    assert eng.demote(u[:20], l[:20]) == 20
    assert len(eng.tier_hot()[0]) == 0
    tier = {(int(a), int(b)) for a, b in zip(u[:20], l[:20])}
    for fn in (eng.get_small, eng.get):
        out, st = fn(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
        hu, hl, lost = eng.tier_hot()
        assert lost == 0 and len(hu) == 20 and {(int(a), int(b)) for a, b in zip(hu, hl)} == tier
    eng.read_records(u, l)                                         # not a get: nothing is logged
    hu, _, lost = eng.tier_hot()
    assert len(hu) == 0 and lost == 0
    reps = 210                                                     # 4 200 tier hits in one call
    out, st = eng.get(np.tile(u[:20], reps), np.tile(l[:20], reps))
    assert (st == E.HIT).all()
    hu, hl, lost = eng.tier_hot(8)
    assert lost == 20 * reps - 4096 and len(hu) == 8
    assert len(eng.tier_hot()[0]) == 0                             # drained
    # what the log names is what promotion takes
    out, st = eng.get_small(u[:20], l[:20])
    hu, hl, _ = eng.tier_hot()
    assert eng.promote(hu, hl) == 20 and eng.host_tier_stats()["records"] == 0
    eng.close()


def test_small_gets_overlap_promotion_and_demotion_without_torn_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 192, 65536
# a demotion of every key fills ~half a lap of the tier, so the ring wraps every other round
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=3 << 30, max_batch=256, host_tier_bytes=16 << 20)
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 78, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
eng.put(u, l, A)
stop = threading.Event(); bad = []; gets = [0]; moved = [0, 0]
def reader():
    while not stop.is_set():
        out, st = eng.get_small(u, l)
        gets[0] += 1
        ok = ((st == E.HIT) & ((out == A).all(axis=1) | (out == B).all(axis=1))) | (st == E.MISS)
        if not ok.all():
            bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
            return
def mover():
    while not stop.is_set():
        moved[0] += eng.demote(u, l)
        moved[1] += eng.promote(u, l)
        if eng.stats()["arena_used"] > 1 << 30:                 # promotion takes fresh arena bytes every time
            eng.compact()
th = [threading.Thread(target=reader) for _ in range(2)] + [threading.Thread(target=mover)]
[t.start() for t in th]
# the main thread rewrites the first half; the second half is left to the mover, so that what one
# demotion sends to the tier is still there when the promotion that follows it runs
h = n // 2
for rnd in range(40):
    eng.put(u[:h], l[:h], (B if rnd % 2 == 0 else A)[:h])
stop.set(); [t.join() for t in th]
assert not bad, bad
ht = eng.host_tier_stats()
assert moved[0] > 0 and moved[1] > 0 and ht["promoted_records"] == moved[1], (moved, ht)
eng.compact()
eng.put(u, l, A)
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
print("no torn pages", gets[0], moved, ht["retired_records"])
'''
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def _drop_in(E, path, hot_rounds, until_promoted=False):
    n, hot = 4096, 256
    cm = E.Cachemap(str(path), 8192, 12, 16)
    assert cm.ok
    pages = np.stack([datagen.make_page("R", 65536, 9000 + c) for c in range(n)])
    nh = np.full(n, 3, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    off = np.arange(n, dtype=np.uint64) << np.uint64(16)
    for base in range(0, n, 256):
        cm.put_batch(off[base:base + 256], nh[base:base + 256], gen[base:base + 256], pages[base:base + 256])
    h = cm.engine_handle()
    assert E.host_tier_stats(h)["records"] > hot
    for _ in range(hot_rounds):
        for i in range(hot):
            assert cm.get(int(off[i]), 3, 0) == pages[i].tobytes(), i
        time.sleep(0.25)                                           # the flusher's round comes within 100 ms
        if until_promoted and E.host_tier_stats(h)["promoted_records"] > 0:
            break
    return cm, h, pages, off, nh, gen


def test_drop_in_promotes_what_gets_read(E, gpu, tmp_path, monkeypatch):
    for k, v in dict(CMB200_ARENA_MB="96", CMB200_SEG_KB="0", CMB200_MAX_BATCH="512", CMB200_PERSIST="0",
                     CMB200_HOST_TIER_MB="1024", CMB200_TIER_PROMOTE="256").items():
        monkeypatch.setenv(k, v)
    (tmp_path / "on").mkdir()
    cm, h, pages, off, nh, gen = _drop_in(E, tmp_path / "on", 20, until_promoted=True)
    for _ in range(3):                                             # two more rounds of reads and promotions
        for i in range(256):
            assert cm.get(int(off[i]), 3, 0) == pages[i].tobytes(), i
        time.sleep(0.25)
    ht = E.host_tier_stats(h)
    assert ht["promoted_records"] > 0, str(ht)
    hits = ht["hits"]
    for i in range(256):
        assert cm.get(int(off[i]), 3, 0) == pages[i].tobytes(), i
    ht2 = E.host_tier_stats(h)
    assert ht2["hits"] - hits <= 8, (str(ht), str(ht2))           # the hot set is read from HBM now
    for base in range(0, 4096, 512):
        out, hit = cm.get_batch(off[base:base + 512], nh[base:base + 512], gen[base:base + 512])
        assert hit.all() and (out == pages[base:base + 512]).all(), base
    st = E.engine_stats(h)
    assert st["entries"] == 4096 and st["dropped_puts"] == 0, st
    cm.free()
    monkeypatch.delenv("CMB200_TIER_PROMOTE")
    (tmp_path / "off").mkdir()
    cm, h, pages, off, nh, gen = _drop_in(E, tmp_path / "off", 1)
    ht = E.host_tier_stats(h)
    assert ht["promoted_records"] == 0 and ht["hits"] > 0, ht
    cm.free()
