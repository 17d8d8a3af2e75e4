"""GPU tests of encryption at rest: k_seal / k_open against the pure-Python ChaCha20-Poly1305 and the
golden vectors; sealed snapshots and chains written and loaded through the engine API with a file key,
checked against tests/snapshot_crypt.py and against the same store saved in the clear; the failure
cases (wrong key, no key, a damaged record, damaged tombstones); and the plaintext-to-sealed migration."""
import hashlib
import json
import os
import random
import struct
import subprocess

import numpy as np
import pytest

import snapshot_crypt as SC

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "chacha20poly1305.json")
H = bytes.fromhex
KEY = bytes(range(0x40, 0x60))
NH = 7


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _msg(case):
    return b"\xff" * case["len"] if case["ff"] else random.Random(case["seed"]).randbytes(case["len"])


def test_batch_equals_golden_at_every_record_size(gpu, E):
    cases = _golden()["records"]
    msgs = [_msg(c) for c in cases]
    # each case has a key of its own, and a batch takes one key: one call per case
    for c, m in zip(cases, msgs):
        out = E.aead_seal_batch(H(c["key"]), [H(c["nonce"])], [H(c["aad"])], [m])[0]
        if "sealed" in c:
            assert out == H(c["sealed"]), c["len"]
        else:
            assert hashlib.sha256(out).hexdigest() == c["sha256"], c["len"]
        back = E.aead_open_batch(H(c["key"]), [H(c["nonce"])], [H(c["aad"])], [out])[0]
        assert back == m
    for v in _golden()["aead"]:
        assert E.aead_seal_batch(H(v["key"]), [H(v["nonce"])], [H(v["aad"])], [H(v["plaintext"])])[0] == H(v["sealed"])


def test_mixed_batch_fills_every_sm_and_flips_reject_one(gpu, E):
    rng = random.Random(11)
    sizes = [0, 1, 15, 16, 17, 63, 64, 65, 24 + 4096] + [rng.randrange(0, 700) for _ in range(3000)]
    sizes += [24 + 65536 + 1024, 24 + (1 << 20) + 1024]
    msgs = [rng.randbytes(n) for n in sizes]
    aads = [rng.randbytes(rng.choice([0, 1, 24, 64, 100])) for _ in sizes]
    nonces = [rng.randbytes(12) for _ in sizes]
    out = E.aead_seal_batch(KEY, nonces, aads, msgs)
    for k in list(range(12)) + rng.sample(range(len(sizes) - 2), 200) + [len(sizes) - 2]:
        assert out[k] == SC.seal(KEY, nonces[k], aads[k], msgs[k]), sizes[k]
    assert out[-1][-16:] == SC.seal(KEY, nonces[-1], aads[-1], msgs[-1])[-16:]
    assert E.aead_open_batch(KEY, nonces, aads, out) == msgs
    # one bit flipped in the ciphertext, the tag or the AAD of three messages: exactly those fail
    bad_out, bad_aad = list(out), list(aads)
    ct_k, tag_k, aad_k = 20, 300, 2000
    b = bytearray(bad_out[ct_k]); b[len(b) // 3 if len(b) > 16 else 0] ^= 0x10; bad_out[ct_k] = bytes(b)
    b = bytearray(bad_out[tag_k]); b[-1] ^= 0x80; bad_out[tag_k] = bytes(b)
    bad_aad[aad_k] = bytes([bad_aad[aad_k][0] ^ 1]) + bad_aad[aad_k][1:] if bad_aad[aad_k] else b"\x01"
    got = E.aead_open_batch(KEY, nonces, bad_aad, bad_out)
    for k, g in enumerate(got):
        assert (g is None) == (k in (ct_k, tag_k, aad_k)), k


# ---- stores ----

def _engines(E, pshift, g, tier=False, n_hint=1200):
    bsize = 1 << pshift
    out = []
    for _ in range(g):
        e = E.Engine(pshift=pshift, accel=1, capacity=4096, arena_bytes=max(n_hint * bsize, 64 << 20),
                     max_batch=256, flags=E.FINGERPRINT)
        if tier:
            e.enable_host_tier(max(n_hint * bsize // 2, 32 << 20))
        out.append(e)
    return out


def _pages(E, pshift, n, seed=5):
    bsize = 1 << pshift
    pages = np.stack([E.gen_chunk_host(seed, c, bsize) for c in range(n)])
    pages[::5] = np.frombuffer(random.Random(seed).randbytes(bsize * len(pages[::5])), np.uint8).reshape(-1, bsize)
    return pages


def _fill(E, engines, pshift, n, tier=False, seed=5):
    """n pages at (NH, 0 .. n-1) with ts 100 + i, split by cmb200_owner; a quarter demoted to the tier."""
    g = len(engines)
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    pages = _pages(E, pshift, n, seed)
    ts = np.arange(100, 100 + n, dtype=np.uint64)
    keys = [E.owner(_fnv(int(a), int(b)), g) for a, b in zip(u, l)]
    for k, e in enumerate(engines):
        idx = np.array([i for i in range(n) if keys[i] == k], dtype=np.int64)
        if len(idx):
            e.put(u[idx], l[idx], pages[idx], ts=ts[idx])
            if tier:
                q = idx[: len(idx) // 4]
                assert e.demote(u[q], l[q]) == len(q)
    return u, l, pages


def _fnv(u, l):
    h = 14695981039346656037
    for b in struct.pack("<QQ", u, l):
        h = ((h ^ b) * 0x100000001B3) & (2**64 - 1)
    return h


def _state(engines, u, l):
    """What a load leaves, per engine: entries, and per address the record, fingerprint, parse
    checkpoints (without word 0, the tag naming where the record lies) and, through cmb200_sample, ts."""
    out = []
    for e in engines:
        words, ok = e.read_checkpoints(u, l)
        fps, fok = e.read_fingerprints(u, l)
        addr, ts, sok = e.sample(np.arange(1 << 14, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        out.append({"entries": e.entries(), "records": e.read_records(u, l), "fp": fps.tolist(), "fp_ok": fok.tolist(),
                    "ckpt_ok": ok.tolist(), "ckpt": words[:, 1:].tolist(),
                    "ts": {(int(a[0]), int(a[1])): int(t) for a, t, k in zip(addr, ts, sok) if k == 1}})
    return out


def _same_state(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        for k in x:
            if k == "ts":
                common = set(x[k]) & set(y[k])
                assert len(common) > 0 and all(x[k][c] == y[k][c] for c in common), (i, k)
            else:
                assert x[k] == y[k], (i, k, next((j for j, (p, q) in enumerate(zip(x[k], y[k])) if p != q), None)
                                      if isinstance(x[k], list) else (x[k], y[k]))


def _close(engines):
    for e in engines:
        e.close()


@pytest.mark.parametrize("pshift", [12, 16, 20])
@pytest.mark.parametrize("g", [1, 2])
def test_sealed_save_decrypts_to_the_plaintext_save_and_loads_the_same(gpu, E, tmp_path, pshift, g):
    n = {12: 1500, 16: 400, 20: 48}[pshift]
    src = _engines(E, pshift, g, tier=True, n_hint=n)
    u, l, _pages_ = _fill(E, src, pshift, n, tier=True)
    handles = [e.h for e in src]
    plain, sealed = str(tmp_path / "plain"), str(tmp_path / "sealed")
    assert E.save_set(handles, plain) == n
    for e in src:
        e.set_file_key(KEY)
    assert E.save_set(handles, sealed) == n
    # the sealed file: the same record stream as the plaintext one, under the key
    _ps, pflags, precs = _read_plain(plain)
    spshift, sflags, chain, srecs = SC.read_base(sealed, KEY)
    assert (spshift, sflags, chain) == (pshift, pflags, 0)
    assert srecs == precs
    raw = open(sealed, "rb").read()
    assert raw[:8] == b"CMB200E1"
    _close(src)
    # loads: the sealed file into keyed engines equals the plaintext file into plain engines
    a, b = _engines(E, pshift, g, n_hint=n), _engines(E, pshift, g, n_hint=n)
    for e in b:
        e.set_file_key(KEY)
    assert E.load_set([e.h for e in a], plain) == n
    assert E.load_set([e.h for e in b], sealed) == n
    _same_state(_state(a, u, l), _state(b, u, l))
    assert all(e.load_rejected() == 0 for e in b)
    _close(a); _close(b)


def _read_plain(path):
    from oracle import snapshot
    return snapshot.read_snapshot(path)


def test_without_a_key_the_file_is_the_plaintext_format(gpu, E, tmp_path):
    from oracle import snapshot
    src = _engines(E, 12, 1, n_hint=300)
    _fill(E, src, 12, 300)
    p = str(tmp_path / "plain")
    E.save_set([src[0].h], p)
    _ps, flags, recs = snapshot.read_snapshot(p)
    q = str(tmp_path / "restated")
    snapshot.write_snapshot(q, 12, recs, bool(flags & 1))
    assert open(p, "rb").read() == open(q, "rb").read()
    _close(src)


def test_wrong_key_and_no_key_store_nothing(gpu, E, tmp_path):
    src = _engines(E, 12, 1, n_hint=300)
    u, l, _ = _fill(E, src, 12, 300)
    src[0].set_file_key(KEY)
    p = str(tmp_path / "sealed")
    E.save_set([src[0].h], p)
    for key in (None, bytes(32)):
        dst = _engines(E, 12, 1, n_hint=300)
        dst[0].set_file_key(key)
        with pytest.raises(RuntimeError):
            E.load_set([dst[0].h], p)
        with pytest.raises(RuntimeError):
            E.load_chain([dst[0].h], p)
        assert dst[0].entries() == 0
        _close(dst)
    # engines of one call with different keys are refused
    other = _engines(E, 12, 1, n_hint=300)
    with pytest.raises(RuntimeError):
        E.save_set([src[0].h, other[0].h], str(tmp_path / "mixed"))
    _close(other); _close(src)


def test_a_flipped_record_bit_drops_that_record_only(gpu, E, tmp_path):
    src = _engines(E, 12, 1, n_hint=300)
    u, l, pages = _fill(E, src, 12, 300)
    src[0].set_file_key(KEY)
    p = str(tmp_path / "sealed")
    E.save_set([src[0].h], p)
    raw = bytearray(open(p, "rb").read())
    # walk to record 17 and flip a bit of its ciphertext
    pos, victim = 80, None
    for k in range(300):
        n = struct.unpack_from("<I", raw, pos)[0]
        if k == 17:
            victim = struct.unpack_from("<QQ", raw, pos + 8)
            raw[pos + 24 + 40] ^= 4
        pos += (n + 48 + 15) & ~15
    open(p, "wb").write(bytes(raw))
    dst = _engines(E, 12, 1, n_hint=300)
    dst[0].set_file_key(KEY)
    assert E.load_set([dst[0].h], p) == 299
    assert dst[0].load_rejected() == 1 and dst[0].entries() == 299
    out, st = dst[0].get(u, l)
    for i in range(300):
        if (int(u[i]), int(l[i])) == victim:
            assert st[i] == E.MISS
        else:
            assert st[i] == E.HIT and (out[i] == pages[i]).all()
    _close(dst); _close(src)


def _tick(E, engines, base, delta):
    E.snapshot_finish(E.chain_begin([e.h for e in engines], base, delta))


def test_sealed_chain_loads_through_load_chain_and_the_loader(gpu, E, tmp_path):
    pshift, n = 12, 800
    src = _engines(E, pshift, 2, n_hint=n)
    for e in src:
        e.set_file_key(KEY)
    u, l, pages = _fill(E, src, pshift, n)
    base = str(tmp_path / "chain")
    _tick(E, src, base, False)
    pages2 = _pages(E, pshift, 100, seed=9)
    g = len(src)
    keys = [E.owner(_fnv(NH, i), g) for i in range(n)]
    for k, e in enumerate(src):
        idx = np.array([i for i in range(100) if keys[i] == k], dtype=np.int64)
        e.put(u[idx], l[idx], pages2[idx], ts=np.full(len(idx), 9999, np.uint64))
        gone = np.array([i for i in range(700, 760) if keys[i] == k], dtype=np.int64)
        e.unset(u[gone], l[gone])
    _tick(E, src, base, True)
    assert open(base + ".d1", "rb").read()[:8] == b"CMB200F1"
    _cid, _k, tombs, recs = SC.read_delta(base + ".d1", KEY)
    assert len(tombs) == 60 and len(recs) == 100 and all(r is not None for r in recs)
    want = pages.copy()
    want[:100] = pages2
    live = np.ones(n, bool)
    live[700:760] = False
    for mode in ("chain", "loader"):
        dst = _engines(E, pshift, 2, n_hint=n)
        for e in dst:
            e.set_file_key(KEY)
        if mode == "chain":
            assert E.load_chain([e.h for e in dst], base) == (n - 60, 1)
        else:
            ld = E.Loader([e.h for e in dst], base)
            while ld.step(97):
                pass
            assert ld.close() == (n - 60, 1)
        got = np.zeros(n, bool)
        for e in dst:
            out, st = e.get(u, l)
            hit = st == E.HIT
            assert (out[hit] == want[hit]).all()
            got |= hit
        assert (got == live).all()
        _close(dst)
    # a flipped bit in the delta's tombstones ends the run before it: the base alone loads
    raw = bytearray(open(base + ".d1", "rb").read())
    raw[80 + 5] ^= 1
    open(base + ".d1", "wb").write(bytes(raw))
    dst = _engines(E, pshift, 2, n_hint=n)
    for e in dst:
        e.set_file_key(KEY)
    assert E.load_chain([e.h for e in dst], base) == (n, 0)
    for e in dst:
        out, st = e.get(u, l)
        hit = st == E.HIT
        assert (out[hit] == pages[hit]).all()
    _close(dst); _close(src)


def test_plaintext_file_with_a_key_loads_and_the_next_base_is_sealed(gpu, E, tmp_path):
    src = _engines(E, 12, 1, n_hint=300)
    u, l, pages = _fill(E, src, 12, 300)
    base = str(tmp_path / "chain")
    _tick(E, src, base, False)
    assert open(base, "rb").read()[:8] == b"CMB200S1"
    dst = _engines(E, 12, 1, n_hint=300)
    dst[0].set_file_key(KEY)
    assert E.load_chain([dst[0].h], base) == (300, 0)
    _tick(E, dst, base, False)
    assert open(base, "rb").read()[:8] == b"CMB200E1"
    _ps, _f, _c, recs = SC.read_base(base, KEY)
    assert len(recs) == 300 and all(r is not None for r in recs)
    _close(dst); _close(src)


def test_snap2lmdb_refuses_a_sealed_base(gpu, E, oracle, tmp_path):
    if oracle.ref() is None:
        pytest.skip("oracle/_ref was not built")
    from test_oracle_pin import _build_snap2lmdb
    exe = _build_snap2lmdb(tmp_path)
    src = _engines(E, 12, 1, n_hint=100)
    _fill(E, src, 12, 100)
    src[0].set_file_key(KEY)
    p = str(tmp_path / "sealed")
    E.save_set([src[0].h], p)
    (tmp_path / "lmdb").mkdir()
    out = subprocess.run([exe, "to-lmdb", p, str(tmp_path / "lmdb"), "2048", "12"], capture_output=True, text=True)
    assert out.returncode != 0 and "encrypted snapshot" in out.stderr
    _close(src)


DROP_IN = """
import os, sys, time
sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
sys.path.insert(0, sys.argv[1])
import datagen
import edge_fuse_b200 as E
d, phase = sys.argv[2], sys.argv[3]
pages = [datagen.make_page("RTZMPAXS"[i % 8], 4096, 7100 + i) for i in range(300)]
cm = E.Cachemap(d, 4096, 12, 12)
if phase == "write":
    for i in range(300):
        cm.put(i << 12, 9, 0, pages[i])
else:
    cm.get(0, 9, 0)                     # the first call starts the engines and, with CMB200_LOAD=background, the load
    while cm.load_progress()[0]:        # the check is of the whole load
        time.sleep(0.05)
    bad = sum(bytes(cm.get(i << 12, 9, 0) or b"") != bytes(pages[i]) for i in range(300))
    print("bad", bad, flush=True)
cm.free()
"""


def _run_drop_in(tmp_path, d, phase, **env_extra):
    import sys
    script = tmp_path / "drive.py"
    script.write_text(DROP_IN)
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_DEVICES="0,0")
    for k in ("CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_LOAD", "CMB200_KEY_FILE"):
        env.pop(k, None)
    env.update(env_extra)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return subprocess.run([sys.executable, str(script), root, str(d), phase], capture_output=True, text=True,
                          timeout=300, env=env)


@pytest.mark.parametrize("load", ["wait", "background"])
def test_drop_in_key_file_across_two_processes(gpu, E, tmp_path, load):
    import datagen
    kf = tmp_path / "key"
    kf.write_text(KEY.hex() + "\n")
    d = tmp_path / "cache"
    d.mkdir()
    w = _run_drop_in(tmp_path, d, "write", CMB200_KEY_FILE=str(kf))
    assert w.returncode == 0, w.stderr[-3000:]
    raw = (d / "cachemap_b200.snap").read_bytes()
    assert raw[:8] == b"CMB200E1"
    # no 64-byte run of any sampled page's plaintext is in the file
    for i in range(0, 300, 7):
        page = bytes(datagen.make_page("RTZMPAXS"[i % 8], 4096, 7100 + i))
        for at in range(0, 4096, 512):
            run = page[at:at + 64]
            if len(set(run)) > 1:
                assert run not in raw, (i, at)
    r = _run_drop_in(tmp_path, d, "read", CMB200_KEY_FILE=str(kf), CMB200_LOAD=load)
    assert r.returncode == 0 and "bad 0" in r.stdout, r.stdout + r.stderr[-3000:]
    # another key: the map starts empty, warns, and leaves the encrypted file as it is
    other = tmp_path / "other"
    other.write_bytes(bytes(32))
    before = (d / "cachemap_b200.snap").read_bytes()
    r = _run_drop_in(tmp_path, d, "read", CMB200_KEY_FILE=str(other), CMB200_LOAD=load)
    assert r.returncode == 0 and "bad 300" in r.stdout and "encrypted" in r.stderr, r.stdout + r.stderr[-3000:]
    assert (d / "cachemap_b200.snap").read_bytes() == before


@pytest.mark.parametrize("name,seed", [("A", 13), ("D", 43)])
def test_seeded_interleavings_during_an_encrypted_background_load(E, gpu, oracle, tmp_path, monkeypatch, name, seed):
    """tests/test_gpu_load_background.py's as-if check of every store operation during a stepped load,
    with every engine holding a file key: the base and its delta are sealed, and the loader opens them."""
    import store_machine as SM
    from test_gpu_load_background import _run_load_machine

    class KeyedEngine(E.Engine):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.set_file_key(KEY)

    cfg = SM.CONFIGS[name]
    for k, v in cfg.environ().items():
        monkeypatch.setenv(k, v)
    monkeypatch.setattr(E, "Engine", KeyedEngine)
    _run_load_machine(E, oracle, cfg, seed, tmp_path)
    base = tmp_path / "cachemap_b200.snap"
    assert base.read_bytes()[:8] == b"CMB200E1" and (tmp_path / "cachemap_b200.snap.d1").read_bytes()[:8] == b"CMB200F1"
