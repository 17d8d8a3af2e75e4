"""GPU tests of the host tier: records demoted from the HBM arena to page-locked, device-mapped host
memory keep their keys, bytes, statuses and counters, and let the drop-in hold the capacity it was
configured with when the records outgrow the arena."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import datagen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need(rec_len):
    return (rec_len + 15) & ~15


def _drop_in_run(E, tmp_path):
    """4096 distinct incompressible 64 KiB pages (~4x the 96 MiB arena) through cachemap_put_batch."""
    cap, n = 8192, 4096
    cm = E.Cachemap(str(tmp_path), cap, 12, 16)
    assert cm.ok
    pages = np.stack([datagen.make_page("R", 65536, 9000 + c) for c in range(n)])
    nh = np.full(n, 3, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    off = np.arange(n, dtype=np.uint64) << np.uint64(16)
    for base in range(0, n, 256):
        cm.put_batch(off[base:base + 256], nh[base:base + 256], gen[base:base + 256], pages[base:base + 256])
    return cm, pages, off, nh, gen


def test_configured_capacity_holds_beyond_the_arena(E, gpu, tmp_path, monkeypatch):
    monkeypatch.setenv("CMB200_ARENA_MB", "96")
    monkeypatch.setenv("CMB200_SEG_KB", "0")
    monkeypatch.setenv("CMB200_MAX_BATCH", "512")
    monkeypatch.setenv("CMB200_PERSIST", "0")
    monkeypatch.setenv("CMB200_HOST_TIER_MB", "1024")
    (tmp_path / "tier").mkdir()
    cm, pages, off, nh, gen = _drop_in_run(E, tmp_path / "tier")
    h = cm.engine_handle()
    st, ht = E.engine_stats(h), E.host_tier_stats(h)
    assert st["entries"] == 4096 and st["dropped_puts"] == 0, st
    assert ht["demoted_records"] > 0 and ht["records"] > 0 and ht["retired_records"] == 0, ht
    rq0, hit0 = cm.counters()
    asked = 0
    for base in range(0, 4096, 512):
        out, hit = cm.get_batch(off[base:base + 512], nh[base:base + 512], gen[base:base + 512])
        assert hit.all() and (out == pages[base:base + 512]).all(), base
        asked += 512
    for i in list(range(0, 4096, 7)) + list(range(64)):
        assert cm.get(int(off[i]), 3, 0) == pages[i].tobytes(), i
        asked += 1
    for base in range(0, 4096, 509):
        k = min(16, 4096 - base)
        got = cm.read_range(3, 0, int(off[base]), k * 65536)
        assert got == pages[base:base + k].tobytes(), base
    rq, hits = cm.counters()
    assert rq == hits and rq - rq0 >= asked and rq - rq0 <= asked + 9 * 16, (rq0, rq, hits, asked)
    assert E.host_tier_stats(h)["hits"] > 0
    cm.free()
    # the control: without a tier, the arena's size decides and most of the early pages are gone
    monkeypatch.delenv("CMB200_HOST_TIER_MB")
    (tmp_path / "plain").mkdir()
    cm, pages, off, nh, gen = _drop_in_run(E, tmp_path / "plain")
    assert E.engine_stats(cm.engine_handle())["entries"] < 4096
    out, hit = cm.get_batch(off[:1024], nh[:1024], gen[:1024])
    assert hit.mean() < 0.5 and (out[hit != 0] == pages[:1024][hit != 0]).all()
    cm.free()


@pytest.mark.parametrize("pshift", [12, 16])
def test_demoted_records_are_the_references_bytes(E, gpu, oracle, pshift):
    bs = 1 << pshift
    kinds = "RTZMPAX"
    n = 70
    pages = np.stack([datagen.make_page(kinds[i % len(kinds)], bs, 300 + i) for i in range(n)])
    for accel in (12, 0):
        eng = E.Engine(pshift=pshift, accel=accel, capacity=4096, arena_bytes=64 << 20, max_batch=64,
                       host_tier_bytes=64 << 20)
        u = np.full(n, 41, dtype=np.uint64)
        l = np.arange(n, dtype=np.uint64)
        eng.put(u, l, pages)
        before = eng.stats()
        extra = np.array([42], dtype=np.uint64)                                          # an absent key
        assert eng.demote(np.concatenate([u, u[:5], extra]), np.concatenate([l, l[:5], extra])) == n
        assert eng.demote(u, l) == 0                                                     # all in the tier already
        after, ht = eng.stats(), eng.host_tier_stats()
        assert after["entries"] == n and ht["records"] == n and ht["demoted_records"] == n
        recs = eng.read_records(u, l)
        for i in range(n):
            blk = pages[i].tobytes() if accel == 0 else oracle.lz4_encode(pages[i], accel)
            want = oracle.record_prefix(int(u[i]), int(l[i]), 0 if accel == 0 else len(blk)) + blk
            assert recs[i] == want, (i, accel)
        assert after["arena_garbage"] - before["arena_garbage"] == sum(_need(len(r)) for r in recs)
        assert ht["demoted_bytes"] == sum(len(r) for r in recs)
        out_b, st_b = eng.get(u, l)
        out_s, st_s = eng.get_small(u, l)
        assert (st_b == E.HIT).all() and (st_s == E.HIT).all()
        assert (out_b == pages).all() and (out_s == pages).all()
        assert eng.host_tier_stats()["hits"] == 2 * n
        eng.close()


def test_overwrite_unset_and_compaction_of_demoted_keys(E, gpu, oracle):
    pshift, bs, n = 12, 4096, 64
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128,
                   host_tier_bytes=16 << 20)
    pages = np.stack([datagen.make_page("TRZM"[i & 3], bs, 500 + i) for i in range(n)])
    newer = np.stack([datagen.make_page("TMRZ"[i & 3], bs, 900 + i) for i in range(8)])
    u = np.full(n, 5, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    lens = eng.put(u, l, pages)
    rec = [_need(24 + (int(c) if c else bs)) for c in lens]
    assert eng.demote(u[:32], l[:32]) == 32
    s0 = eng.stats()
    assert s0["arena_garbage"] == sum(rec[:32])
    lens8 = eng.put(u[:8], l[:8], newer)                       # overwrite demoted keys: new records in the arena
    eng.unset(u[8:16], l[8:16])                                # unset demoted keys
    s1, ht = eng.stats(), eng.host_tier_stats()
    assert s1["entries"] == n - 8
    assert s1["arena_garbage"] == sum(rec[:32])                # nothing in the arena was replaced
    assert ht["garbage"] == sum(rec[:16]) and ht["records"] == 16
    want = pages.copy()
    want[:8] = newer
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st[8:16] == E.MISS).all()
        live = np.r_[0:8, 16:n]
        assert (st[live] == E.HIT).all() and (out[live] == want[live]).all()
    got = eng.compact()
    s2, ht2 = eng.stats(), eng.host_tier_stats()
    assert got > 0 and s2["arena_garbage"] == 0 and s2["entries"] == n - 8
    assert s2["arena_used"] == sum(rec[32:]) + sum(_need(24 + int(c)) for c in lens8)
    assert ht2["records"] == 16 and ht2["garbage"] == ht["garbage"]
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert (st[live] == E.HIT).all() and (out[live] == want[live]).all() and (st[8:16] == E.MISS).all()
    eng.close()


def test_wrap_around_retires_the_oldest_records(E, gpu):
    pshift, bs, n = 12, 4096, 300
    tier = 256 << 10                                           # ~62 incompressible records per lap
    eng = E.Engine(pshift=pshift, accel=12, capacity=4096, arena_bytes=64 << 20, max_batch=128,
                   host_tier_bytes=tier)
    pages = np.stack([datagen.make_page("R", bs, 700 + i) for i in range(n)])
    u = np.full(n, 6, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    eng.put(u, l, pages)
    for base in range(0, n, 50):
        assert eng.demote(u[base:base + 50], l[base:base + 50]) == 50
    for fn in (eng.get, eng.get_small):
        out, st = fn(u, l)
        assert ((st == E.HIT) | (st == E.MISS)).all(), np.unique(st)
        hit = st == E.HIT
        assert (out[hit] == pages[hit]).all()
        assert hit[-50:].all() and not hit[:50].any()          # newest demoted live, oldest retired
        assert eng.entries() == int(hit.sum())
    ht = eng.host_tier_stats()
    assert ht["retired_records"] == n - eng.entries() and ht["records"] == eng.entries()
    assert ht["used"] <= ht["bytes"] == tier
    # the engine keeps working after the wrap: retired keys can be put again
    eng.put(u[:50], l[:50], pages[:50])
    out, st = eng.get_small(u[:50], l[:50])
    assert (st == E.HIT).all() and (out == pages[:50]).all()
    eng.close()


def test_small_gets_overlap_demotion_and_wrap_without_torn_pages(E, gpu):
    code = r'''
import sys, os, threading
sys.path.insert(0, os.getcwd())
import numpy as np, edge_fuse_b200 as E
n, bs = 192, 65536
eng = E.Engine(pshift=16, accel=12, capacity=8192, arena_bytes=3 << 30, max_batch=256, host_tier_bytes=4 << 20)
# two contents per key (records of different sizes); one demotion call of all keys laps the tier
A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
u = np.full(n, 77, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
eng.put(u, l, A)
stop = threading.Event(); bad = []; gets = [0]; demoted = [0]
def reader():
    while not stop.is_set():
        out, st = eng.get_small(u, l)
        gets[0] += 1
        ok = ((st == E.HIT) & ((out == A).all(axis=1) | (out == B).all(axis=1))) | (st == E.MISS)
        if not ok.all():
            bad.append((int((~ok).sum()), st[~ok][:4].tolist()))
            return
def demoter():
    while not stop.is_set():
        demoted[0] += eng.demote(u, l)
th = [threading.Thread(target=reader) for _ in range(2)] + [threading.Thread(target=demoter)]
[t.start() for t in th]
for rnd in range(40):
    eng.put(u, l, B if rnd % 2 == 0 else A)
stop.set(); [t.join() for t in th]
assert not bad, bad
ht = eng.host_tier_stats()
assert demoted[0] > 0 and ht["retired_records"] > 0, (demoted, ht)
eng.put(u, l, A)
out, st = eng.get_small(u, l)
assert (st == E.HIT).all() and (out == A).all()
print("no torn pages", gets[0], demoted[0], ht["retired_records"])
'''
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "no torn pages" in out.stdout, out.stdout + out.stderr


def test_snapshot_of_both_tiers_loads_anywhere(E, gpu, tmp_path):
    n, bs = 1000, 65536
    pages = np.stack([datagen.make_page("RTZMPAX"[i % 7], bs, 1100 + i) for i in range(n)])
    u = np.full(n, 8, dtype=np.uint64)
    l = np.arange(n, dtype=np.uint64)
    geo = dict(pshift=16, accel=12, capacity=4096, arena_bytes=16 << 20, max_batch=128)
    eng = E.Engine(host_tier_bytes=256 << 20, **geo)
    for base in range(0, n, 100):                              # the arena holds ~ 300 of these pages
        eng.put(u[base:base + 100], l[base:base + 100], pages[base:base + 100], ts=np.arange(base, base + 100, dtype=np.uint64))
        if base < n - 200:
            assert eng.demote(u[base:base + 100], l[base:base + 100]) == 100
            eng.compact()
    assert eng.stats()["dropped_puts"] == 0 and eng.host_tier_stats()["records"] == n - 200
    recs = eng.read_records(u, l)
    path = str(tmp_path / "both.snap")
    assert eng.save(path) == n
    eng.close()
    for e2 in (E.Engine(host_tier_bytes=256 << 20, **geo), E.Engine(**dict(geo, arena_bytes=512 << 20))):
        assert e2.load(path) == n and e2.entries() == n and e2.stats()["dropped_puts"] == 0
        assert (e2.host_tier_stats()["demoted_records"] > 0) == (e2.stats()["arena_bytes"] < 32 << 20)
        assert e2.read_records(u, l) == recs
        for fn in (e2.get, e2.get_small):
            out, st = fn(u, l)
            assert (st == E.HIT).all() and (out == pages).all()
        e2.close()


def test_multi_gpu_calls_refuse_a_tiered_engine(E, gpu):
    L = E.lib()
    eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64, host_tier_bytes=1 << 20)
    pages = np.stack([datagen.make_page("T", 4096, i) for i in range(8)])
    u = np.full(8, 9, dtype=np.uint64)
    l = np.arange(8, dtype=np.uint64)
    eng.put(u, l, pages)
    eng.demote(u[:4], l[:4])
    before, ht = eng.stats(), eng.host_tier_stats()
    h = eng.h
    buf = (ctypes.c_uint8 * 64)()
    size = ctypes.c_uint64(0)
    t = ctypes.c_uint64(0)
    assert L.cmb200_set_stream_order(h, 100, 2) == -1 and "host tier" in E.last_error()
    assert L.cmb200_put_step(h, 0, None, None, None, 0, None, 0, None, None, ctypes.byref(t)) == -1
    assert L.cmb200_import_records_dev(h, 0, None, 0) == -1
    assert L.cmb200_arena_ipc_handle(h, buf, ctypes.byref(size)) == -1
    assert L.cmb200_open_peer(h, 0, buf, 0) == -1
    assert L.cmb200_host_tier_enable(h, 1 << 20) == -1                   # once only
    after = eng.stats()
    for k in ("entries", "put_chunks", "arena_used", "arena_garbage", "remote_entries"):
        assert after[k] == before[k], k
    assert eng.host_tier_stats() == ht
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.close()
    # and the other way round: no tier after a multi-GPU call, nor after the first put
    e2 = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    e2.set_stream_order(1, 1)
    assert L.cmb200_host_tier_enable(e2.h, 1 << 20) == -1
    e2.close()
    e3 = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    e3.put(u, l, pages)
    assert L.cmb200_host_tier_enable(e3.h, 1 << 20) == -1
    assert e3.host_tier_stats()["bytes"] == 0
    e3.close()
