"""One map over several engines (CMB200_DEVICES) on the GPU.  Every test runs with two engines on one
H100 ("0,0": the routing, the per-engine rings and queues, the snapshot set and the page moves without a
peer copy) and, where the machine has two GPUs or more, with every device ("all": the same through
cudaMemcpyPeerAsync).  With one GPU the second case is skipped: cross-device copies are not exercised
there."""
import json
import os
import re
import shutil
import struct
import subprocess
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def fnv1a64(data: bytes) -> int:
    h = 0xcbf29ce484222325
    for b in data:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def owner_of(u: int, l: int, g: int) -> int:
    key = fnv1a64(struct.pack("<QQ", u, l))
    return ((key >> 32) * g) >> 32


@pytest.fixture(params=["0,0", "all"])
def devices(request, gpu):
    if request.param == "all" and gpu < 2:
        pytest.skip("one GPU: cross-device peer copies need two")
    return request.param


def _engines_expected(E, devices):
    return E.device_count() if devices == "all" else len(devices.split(","))


@pytest.mark.gpu
def test_drop_in_c_caller_over_engines(E, devices, tmp_path):
    """The unchanged tests/c/drop_in_test.c (async puts, read-back, counters, ranges, checkpoint, a
    second map on the same directory) against a map of several engines."""
    exe = tmp_path / "drop_in_test"
    lib_dir = os.path.dirname(E.library_path())
    subprocess.run(["gcc", "-std=c99", "-D_DEFAULT_SOURCE", "-O2", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c", "drop_in_test.c"), "-L", lib_dir, "-lcachemap",
                    f"-Wl,-rpath,{lib_dir}", "-o", str(exe)], check=True)
    env = dict(os.environ, CMB200_ARENA_MB="512", CMB200_MAX_BATCH="512", CMB200_DEVICES=devices)
    for pshift, n in ((15, 300), (16, 200), (12, 500)):
        store = tmp_path / f"store{pshift}"
        store.mkdir()
        out = subprocess.run([str(exe), str(store), str(pshift), str(n)], capture_output=True, text=True, env=env,
                             timeout=300)
        assert out.returncode == 0, (pshift, out.returncode, out.stdout, out.stderr)
        assert "drop_in_test ok" in out.stdout and "ratio:" in out.stdout


@pytest.mark.gpu
def test_exerciser_hit_ratios_over_engines(E, devices, tmp_path):
    """The unchanged tests/c/exerciser.c (capacity == count, one eviction per put once full): the hit
    ratio of every phase within 2 points of the reference's (tests/golden/ref_exerciser.json), with the
    eviction decision taken over all engines."""
    gold = json.load(open(os.path.join(GOLD, "ref_exerciser.json")))
    lib_dir = os.path.join(ROOT, "edge_fuse_b200")
    exe = str(tmp_path / "exer")
    subprocess.check_call(["gcc", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c", "exerciser.c"),
                           "-o", exe, "-L", lib_dir, "-lcachemap", f"-Wl,-rpath,{lib_dir}", "-lpthread"])
    n = gold["objects"]
    ours = []
    for r in gold["runs"]:
        d = tmp_path / f"exer{r['seed']}"
        d.mkdir()
        env = dict(os.environ, CMB200_ARENA_MB="2048", CMB200_PERSIST="0", CMB200_DEVICES=devices)
        out = subprocess.run([exe, str(d), str(n), str(gold["pshift"]), str(r["seed"])], capture_output=True, text=True,
                             timeout=300, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        got = {m.group(1): int(m.group(2)) / int(m.group(3)) for m in re.finditer(r"phase (\w+) hits (\d+) of (\d+)", out.stdout)}
        ent = [int(x) for x in re.findall(r"entries_after_\w+ (\d+)", out.stdout)]
        # nothing is evicted below capacity, whichever flusher decides
        assert len(got) == 5 and got["read1"] == 1.0 and got["read2"] == 1.0, out.stdout
        assert ent[0] == n and n - 64 <= ent[1] <= n, ent
        ours.append(got)
    for phase in ("reput_new", "reput_old", "read4"):
        a = 100 * float(np.mean([g[phase] for g in ours]))
        b = 100 * float(np.mean([h / t for h, t in (r["phases"][phase] for r in gold["runs"])]))
        assert abs(a - b) <= 2.0, (phase, a, b)


def _pages(E, n, bsize, seed):
    return np.stack([E.gen_chunk_host(seed, c, bsize) for c in range(n)])


def _ckpt_count(E, handles, u, l):
    return sum(int((E.read_checkpoints(h, u, l)[1] == 1).sum()) for h in handles)


@pytest.mark.gpu
def test_snapshot_moves_between_engine_counts(E, devices, tmp_path, monkeypatch):
    """A directory saved by G engines is one file in the usual format (oracle/snapshot.py reads it);
    it loads into 1 and into 3 engines with every page, the same entries and the parse checkpoints."""
    from oracle import snapshot
    monkeypatch.setenv("CMB200_ARENA_MB", "256")
    monkeypatch.delenv("CMB200_HOST_TIER_MB", raising=False)
    monkeypatch.delenv("CMB200_PERSIST", raising=False)
    monkeypatch.setenv("CMB200_DEVICES", devices)
    n, ps = 3000, 12
    pages = _pages(E, n, 1 << ps, 11)
    off = np.arange(n, dtype=np.uint64) << np.uint64(ps)
    nh = np.full(n, 4242, dtype=np.uint64)
    gen = np.ones(n, dtype=np.uint32)
    u, l = nh, (off >> np.uint64(ps)) | (np.uint64(1) << np.uint64(44))
    store = tmp_path / "store"
    store.mkdir()
    cm = E.Cachemap(str(store), 8192, 12, ps)
    cm.put_batch(off, nh, gen, pages)
    hs = cm.engine_handles()
    assert len(hs) == _engines_expected(E, devices)
    per = [E.engine_stats(h)["entries"] for h in hs]
    assert sum(per) == n and min(per) > 0, per
    ckpts = _ckpt_count(E, hs, u, l)
    assert ckpts > 0
    assert cm.checkpoint() == 0
    cm.free()
    snap = store / "cachemap_b200.snap"
    pshift, _, recs = snapshot.read_snapshot(str(snap))
    assert pshift == ps and len(recs) == n
    assert {struct.unpack("<QQ", r[3][:16]) for r in recs} == set(zip(u.tolist(), l.tolist()))
    saved = tmp_path / "saved.snap"
    shutil.copy(snap, saved)
    for g_new in ("0", "0,0,0"):
        shutil.copy(saved, snap)
        monkeypatch.setenv("CMB200_DEVICES", g_new)
        cm = E.Cachemap(str(store), 8192, 12, ps)
        out, hit = cm.get_batch(off, nh, gen)
        hs = cm.engine_handles()
        assert len(hs) == len(g_new.split(","))
        assert hit.all() and (out == pages).all(), g_new
        ent = [E.engine_stats(h)["entries"] for h in hs]
        assert sum(ent) == n and min(ent) > 0, (g_new, ent)
        for k, h in enumerate(hs):         # every key on its owner
            _, ok = E.read_checkpoints(h, u, l)
            mine = np.array([owner_of(int(a), int(b), len(hs)) == k for a, b in zip(u, l)])
            assert ((ok >= 0) == mine).all(), (g_new, k)
        assert _ckpt_count(E, hs, u, l) == ckpts, g_new
        cm.free()


@pytest.mark.gpu
def test_host_tier_on_every_engine(E, devices, tmp_path, monkeypatch):
    """A small arena per engine and a host tier: four arenas' worth of incompressible pages all stay,
    and every engine demoted some of its own."""
    monkeypatch.setenv("CMB200_DEVICES", devices)
    monkeypatch.setenv("CMB200_ARENA_MB", "64")
    monkeypatch.setenv("CMB200_HOST_TIER_MB", "1024")
    monkeypatch.setenv("CMB200_PERSIST", "0")
    g = _engines_expected(E, devices)
    bs = 65536
    n = 4 * g * (64 << 20) // bs
    rng = np.random.default_rng(3)
    pages = rng.integers(0, 256, (n, bs), dtype=np.uint8)
    off = np.arange(n, dtype=np.uint64) << np.uint64(16)
    nh = np.full(n, 99, dtype=np.uint64)
    gen = np.zeros(n, dtype=np.uint32)
    cm = E.Cachemap(str(tmp_path), 4 * n, 12, 16)
    for at in range(0, n, 1024):
        cm.put_batch(off[at:at + 1024], nh[at:at + 1024], gen[at:at + 1024], pages[at:at + 1024])
    out, hit = cm.get_batch(off, nh, gen)
    assert hit.all() and (out == pages).all()
    hs = cm.engine_handles()
    assert len(hs) == g
    assert sum(E.engine_stats(h)["entries"] for h in hs) == n
    for h in hs:
        t = E.host_tier_stats(h)
        assert t["demoted_records"] > 0 and t["retired_records"] == 0, t
    cm.free()


@pytest.mark.gpu
def test_single_gets_overlap_puts_without_torn_pages(E, devices, tmp_path, monkeypatch):
    """Two reader threads of cachemap_get against a writer that rewrites keys of every engine with
    pages of two contents: each page a get returns is one of the two pages of its key, whole.  (A get
    that overlaps the rewrite of its key can miss; that happens with one engine as well.)"""
    monkeypatch.setenv("CMB200_DEVICES", devices)
    monkeypatch.setenv("CMB200_ARENA_MB", "1024")
    monkeypatch.setenv("CMB200_PERSIST", "0")
    n, bs = 128, 65536
    A = np.stack([E.gen_chunk_host(5, 8 * c + 1, bs) for c in range(n)])
    B = np.stack([E.gen_chunk_host(5, 8 * c + 3, bs) for c in range(n)])
    off = np.arange(n, dtype=np.uint64) << np.uint64(16)
    nh = np.full(n, 77, dtype=np.uint64)
    gen = np.ones(n, dtype=np.uint32)
    g = _engines_expected(E, devices)
    owners = {owner_of(77, i | (1 << 44), g) for i in range(n)}
    assert owners == set(range(g))
    cm = E.Cachemap(str(tmp_path), 8192, 12, 16)
    cm.put_batch(off, nh, gen, A)
    stop = threading.Event()
    bad, gets = [], [0]

    def reader(seed):
        rng = np.random.default_rng(seed)
        while not stop.is_set():
            i = int(rng.integers(0, n))
            p = cm.get(int(off[i]), 77, 1)
            gets[0] += 1
            if p is None:
                continue
            q = np.frombuffer(p, dtype=np.uint8)
            if not ((q == A[i]).all() or (q == B[i]).all()):
                bad.append((i, "torn"))
                return

    th = [threading.Thread(target=reader, args=(s,)) for s in range(2)]
    [t.start() for t in th]
    for rnd in range(30):
        cm.put_batch(off, nh, gen, B if rnd % 2 == 0 else A)
    stop.set()
    [t.join() for t in th]
    assert not bad, bad
    assert gets[0] > 0
    out, hit = cm.get_batch(off, nh, gen)
    assert hit.all() and (out == A).all()
    cm.free()


@pytest.mark.gpu
def test_device_pages_round_trip(E, devices, tmp_path, monkeypatch):
    """cachemap_put_batch_dev / cachemap_get_batch_dev with the pages on the first device: each engine's
    pages are gathered, (peer-)copied and scattered by k_move_pages; the pages come back where they
    were, and a miss leaves its page of the output untouched."""
    monkeypatch.setenv("CMB200_DEVICES", devices)
    monkeypatch.setenv("CMB200_ARENA_MB", "512")
    monkeypatch.setenv("CMB200_PERSIST", "0")
    L = E.lib()
    n, bs = 1000, 16384
    pages = _pages(E, n, bs, 21)
    off = np.arange(n, dtype=np.uint64) << np.uint64(14)
    nh = np.full(n, 555, dtype=np.uint64)
    gen = np.full(n, 2, dtype=np.uint32)
    cm = E.Cachemap(str(tmp_path), 8192, 12, 14)
    h0 = cm.engine_handle()
    assert len(cm.engine_handles()) == _engines_expected(E, devices)
    src = L.cmb200_dev_alloc(h0, n * bs)
    dst = L.cmb200_dev_alloc(h0, (n + 10) * bs)
    try:
        assert L.cmb200_memcpy_h2d(h0, src, pages.ctypes.data, n * bs) == 0
        cm.put_batch(off, nh, gen, src, on_dev=True)
        # 10 addresses never put among the requests: misses
        qoff = np.concatenate([off, (np.arange(10, dtype=np.uint64) + np.uint64(n)) << np.uint64(14)])
        qnh = np.full(n + 10, 555, dtype=np.uint64)
        qgen = np.full(n + 10, 2, dtype=np.uint32)
        perm = np.random.default_rng(4).permutation(n + 10)
        qoff, qnh, qgen = qoff[perm], qnh[perm], qgen[perm]
        sentinel = np.full((n + 10, bs), 0xA5, dtype=np.uint8)
        assert L.cmb200_memcpy_h2d(h0, dst, sentinel.ctypes.data, (n + 10) * bs) == 0
        _, hit = cm.get_batch(qoff, qnh, qgen, out=dst, on_dev=True)
        back = np.empty((n + 10, bs), dtype=np.uint8)
        assert L.cmb200_memcpy_d2h(h0, back.ctypes.data, dst, (n + 10) * bs) == 0
        for j, p in enumerate(perm):
            if p < n:
                assert hit[j] == 1 and (back[j] == pages[p]).all(), j
            else:
                assert hit[j] == 0 and (back[j] == 0xA5).all(), j
        assert cm.counters() == (n + 10, n)
    finally:
        L.cmb200_dev_free(h0, src)
        L.cmb200_dev_free(h0, dst)
    cm.free()


@pytest.mark.gpu
def test_move_pages_gathers_and_scatters(E, gpu):
    """cmb200_move_pages alone: dst[dst_idx[i]] = src[src_idx[i]] for a random permutation, and the
    plain contiguous copy."""
    L = E.lib()
    eng = E.Engine(pshift=12, accel=12, capacity=1024, arena_bytes=16 << 20, max_batch=64)
    n, bs = 777, 4096
    pages = _pages(E, n, bs, 31)
    src, dst = eng.dev_alloc(n * bs), eng.dev_alloc(n * bs)
    try:
        eng.h2d(src, pages)
        rng = np.random.default_rng(8)
        si, di = rng.permutation(n).astype(np.uint32), rng.permutation(n).astype(np.uint32)
        eng.move_pages(n, dst, src, dst_idx=di, src_idx=si)
        back = np.empty_like(pages)
        eng.d2h(back, dst)
        assert (back[di] == pages[si]).all()
        eng.move_pages(n, dst, src)
        eng.d2h(back, dst)
        assert (back == pages).all()
        assert L.cmb200_move_pages(eng.h, 1, dst + 8, None, src, None) != 0     # 16-byte alignment is required
    finally:
        eng.dev_free(src)
        eng.dev_free(dst)
        eng.close()
