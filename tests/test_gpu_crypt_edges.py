"""GPU tests of encryption at rest at its edges, each checked against tests/snapshot_crypt.py (SC):

  A. k_seal / k_open at the lane and group boundaries of text and AAD, and one-bit flips that must fail
     exactly the flipped message;
  B. Poly1305 driven to chosen accumulator values (tests/crypt_edges.py's target_message), and long
     all-0xff ciphertexts under an r with many bits set;
  C. sealed saves that span several windows of the writer and both engines' sections;
  D. deltas whose tombstone blocks give lanes a second group, GPU-written and written by
     crypt_edges.write_delta;
  E. files the GPU did not write, records whose tag is authentic but whose compressed_length is not,
     records moved between ordinals or files, through load_set, load_chain and the Loader;
  F. loads into engines whose max_batch stages one record at a time.

No test hands k_restore a record that a correct k_open refuses: every rejection is asserted before any
get touches its address."""
import random
import struct

import numpy as np
import pytest

import crypt_edges as CE
import snapshot_crypt as SC
from test_gpu_snapshot_crypt import KEY, _close, _fnv

pytestmark = pytest.mark.gpu

NH = 11


def _flip(b: bytes, at: int, bit: int = 1) -> bytes:
    x = bytearray(b)
    x[at] ^= bit
    return bytes(x)


# ---- A. the kernels against the pure-Python AEAD at lane and group boundaries ----

BOUNDARY = list(range(0, 321)) + [2048 * k + d for k in range(1, 5) for d in (-17, -16, -1, 0, 1, 15, 16, 17)]


def _check_batch(E, nonces, aads, msgs):
    """Seal equals SC.seal, open gives the plaintext back, and one-bit flips in the last AAD group, in a
    lane's second text group and in the tag's first and last bytes fail exactly the flipped messages."""
    out = E.aead_seal_batch(KEY, nonces, aads, msgs)
    for k in range(len(msgs)):
        assert out[k] == SC.seal(KEY, nonces[k], aads[k], msgs[k]), (k, len(aads[k]), len(msgs[k]))
    assert E.aead_open_batch(KEY, nonces, aads, out) == msgs
    n = len(msgs)
    rounds = [
        ("last AAD group", [k for k in range(n) if aads[k] and k % 2 == 0], lambda k, a, s: (_flip(a, len(a) - 1 - (k % min(64, len(a))), 0x80), s)),
        ("second text group", [k for k in range(n) if len(msgs[k]) > 2048 and k % 2 == 1],
         lambda k, a, s: (a, _flip(s, 2048 + k % (len(msgs[k]) - 2048), 0x04))),
        ("tag byte 0", list(range(0, n, 3)), lambda k, a, s: (a, _flip(s, len(s) - 16, 0x01))),
        ("tag byte 15", list(range(1, n, 3)), lambda k, a, s: (a, _flip(s, len(s) - 1, 0x80))),
    ]
    for name, ks, bend in rounds:
        assert ks, name
        bad_a, bad_s = list(aads), list(out)
        for k in ks:
            bad_a[k], bad_s[k] = bend(k, aads[k], out[k])
        got = E.aead_open_batch(KEY, nonces, bad_a, bad_s)
        flipped = set(ks)
        for k, g in enumerate(got):
            assert (g is None) == (k in flipped), (name, k, len(aads[k]), len(msgs[k]))


def test_every_text_length_at_lane_and_group_boundaries(gpu, E):
    rng = random.Random(1)
    msgs = [rng.randbytes(n) for n in BOUNDARY]
    aads = [rng.randbytes(rng.choice([0, 13, 24])) for _ in msgs]
    nonces = [rng.randbytes(12) for _ in msgs]
    _check_batch(E, nonces, aads, msgs)


def test_every_aad_length_at_lane_and_group_boundaries(gpu, E):
    rng = random.Random(2)
    aad_lens = BOUNDARY + [0, 24, 64, 65537]
    msgs, aads = [], []
    for j, a in enumerate(aad_lens):
        for t in (0, 24 + 40, 2048 + 17 + (j % 3) * 16):
            msgs.append(rng.randbytes(t))
            aads.append(rng.randbytes(a))
    nonces = [rng.randbytes(12) for _ in msgs]
    _check_batch(E, nonces, aads, msgs)


# ---- B. Poly1305 at chosen accumulator values ----

def test_poly1305_reaches_every_chosen_residue(gpu, E):
    rng = random.Random(3)
    cases = []
    positions = [(p, a) for p in CE.TARGET_PREFIXES for a in CE.TARGET_AADS]
    for T in CE.SMALL_TARGETS:
        for j in range(72):                        # at least 64 per residue, spread over every position
            cases.append((str(T), T, *positions[j % len(positions)]))
    for name, t in CE.EDGE_TARGETS:
        for p, a in positions:
            cases.append((name, t, p, a))
    nonces, aads, msgs, cts, tags = [], [], [], [], []
    for name, t, prefix, aad_len in cases:
        aad = rng.randbytes(aad_len)
        nonce, pt, ct, T = CE.find_target(KEY, aad, prefix, t, rng)
        _r, s = CE.poly_rs(KEY, nonce)
        nonces.append(nonce); aads.append(aad); msgs.append(pt); cts.append(ct)
        tags.append(((T + s) & CE.M128).to_bytes(16, "little"))
    out = E.aead_seal_batch(KEY, nonces, aads, msgs)
    for k, (name, _t, prefix, aad_len) in enumerate(cases):
        assert out[k] == cts[k] + tags[k], (name, prefix, aad_len)
        assert out[k] == SC.seal(KEY, nonces[k], aads[k], msgs[k])
    assert E.aead_open_batch(KEY, nonces, aads, out) == msgs
    # every single-byte change of each tag fails, and only that message
    for at in range(16):
        bad = [o[:len(o) - 16 + at] + bytes([o[len(o) - 16 + at] ^ (1 + (k + at) % 255)]) + o[len(o) - 15 + at:]
               for k, o in enumerate(out)]
        assert all(g is None for g in E.aead_open_batch(KEY, nonces, aads, bad)), at


def test_all_ff_ciphertexts_under_a_dense_r(gpu, E):
    nonce, bits = CE.best_r_nonce(KEY)
    assert bits >= 70                  # a random r has about 53 of its 106 free bits set
    lens = [16, 64, 2048, 2064, 4096 + 24, 8192 + 16, 24 + 65536 + 1024, 24 + (1 << 20) + 1024]
    msgs, aads = [], []
    for n in lens:
        for a in (0, 16, 2064):
            msgs.append(SC.chacha20(KEY, 1, nonce, b"\xff" * n))
            aads.append(b"\xff" * a)
    nonces = [nonce] * len(msgs)
    out = E.aead_seal_batch(KEY, nonces, aads, msgs)
    for k, o in enumerate(out):
        assert o[:-16] == b"\xff" * len(msgs[k])
        assert o == SC.seal(KEY, nonce, aads[k], msgs[k]), (len(msgs[k]), len(aads[k]))
    assert E.aead_open_batch(KEY, nonces, aads, out) == msgs


# ---- stores ----

def _mk(E, pshift, g, n, key=None, tier=False, max_batch=256, flags=None, small=False):
    """g engines for n records; small: records of near-zero pages, a few dozen bytes each."""
    bsize = 1 << pshift
    arena = max((n // g + 64) * (64 if small else bsize + 64), 64 << 20)
    out = []
    for _ in range(g):
        e = E.Engine(pshift=pshift, accel=1, capacity=max(4096, 2 * n), arena_bytes=arena, max_batch=max_batch,
                     flags=E.FINGERPRINT if flags is None else flags)
        if tier:
            e.enable_host_tier(max(arena // 2, 32 << 20))
        if key is not None:
            e.set_file_key(key)
        out.append(e)
    return out


def _small_pages(ids, bsize):
    """Near-zero pages stamped with their id, and every fourth a self-repeating page: both compress to a
    few dozen bytes."""
    ids = np.asarray(ids, dtype=np.uint64)
    pages = np.zeros((len(ids), bsize), np.uint8)
    pages[:, :8] = ids.view(np.uint8).reshape(-1, 8)
    rep = (ids % np.uint64(4)) == 0
    if rep.any():
        pat = np.frombuffer(b"abcdefgh" * 4, np.uint8)
        pages[rep, 8:] = np.tile(pat, bsize // 32 + 1)[:bsize - 8]
    return pages


def _random_pages(ids, bsize, seed=0):
    out = np.empty((len(ids), bsize), np.uint8)
    for k, i in enumerate(ids):
        out[k] = np.frombuffer(random.Random(seed * 1_000_003 + int(i)).randbytes(bsize), np.uint8)
    return out


def _owner_split(E, u, l, g):
    keys = np.array([E.owner(_fnv(int(a), int(b)), g) for a, b in zip(u, l)])
    return [np.nonzero(keys == k)[0] for k in range(g)]


def _put(E, engines, u, l, page_fn, ts=None, chunk=16384, tier=False):
    """Puts page_fn(index array) at (u, l) by owner, in chunks; a quarter of each engine's records
    demoted to its host tier."""
    ts = np.arange(100, 100 + len(u), dtype=np.uint64) if ts is None else ts
    for e, idx in zip(engines, _owner_split(E, u, l, len(engines))):
        for c0 in range(0, len(idx), chunk):
            q = idx[c0:c0 + chunk]
            e.put(u[q], l[q], page_fn(q), ts=ts[q])
        if tier:
            d = idx[: len(idx) // 4]
            for c0 in range(0, len(d), chunk):
                assert e.demote(u[d[c0:c0 + chunk]], l[d[c0:c0 + chunk]]) == len(d[c0:c0 + chunk])


def _same_load(a, b, u, l, bsize, fp=True, samples=1 << 14, what=None):
    """_state / _same_state of two loads, read in slices so that a large store stays small in memory
    (fp: the engines keep fingerprints; samples: cmb200_sample draws for the timestamps)."""
    chunk = max(8, (64 << 20) // (bsize + 1048))
    for ea, eb in zip(a, b):
        assert ea.entries() == eb.entries(), what
    for c0 in range(0, len(u), chunk):
        uu, ll = u[c0:c0 + chunk], l[c0:c0 + chunk]
        for i, (ea, eb) in enumerate(zip(a, b)):
            assert ea.read_records(uu, ll) == eb.read_records(uu, ll), (what, i, c0)
            if fp:
                fa, oa = ea.read_fingerprints(uu, ll)
                fb, ob = eb.read_fingerprints(uu, ll)
                # a fingerprint is defined only where the engine holds the record (ok == 1)
                bad = (oa != ob) | ((oa == 1) & (fa != fb).any(1))
                assert not bad.any(), (what, i, c0, np.nonzero(bad)[0][:5])
            wa, ka = ea.read_checkpoints(uu, ll)
            wb, kb = eb.read_checkpoints(uu, ll)
            assert (ka == kb).all() and (wa[ka == 1, 1:] == wb[kb == 1, 1:]).all(), (what, i, c0)
    r = np.arange(samples, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    for ea, eb in zip(a, b):
        xa, ta, sa = ea.sample(r)
        xb, tb, sb = eb.sample(r)
        A = {(int(p[0]), int(p[1])): int(t) for p, t, k in zip(xa, ta, sa) if k == 1}
        B = {(int(p[0]), int(p[1])): int(t) for p, t, k in zip(xb, tb, sb) if k == 1}
        common = set(A) & set(B)
        assert common and all(A[c] == B[c] for c in common), what


def _read_plain(path):
    from oracle import snapshot
    return snapshot.read_snapshot(path)


# ---- C. saves that span several windows ----

@pytest.mark.parametrize("pshift,n", [(12, 140000), (16, 2300), (20, 160)])
def test_sealed_save_across_windows_and_sections(gpu, E, tmp_path, pshift, n):
    bsize = 1 << pshift
    small = pshift == 12
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    split = _owner_split(E, u, l, 2)
    if small:
        # more than a window's 65 536 records on engine 0, a few thousand on engine 1
        keep = np.sort(np.concatenate([split[0], split[1][:3000]]))
        u, l, n = u[keep], l[keep], len(keep)
        split = _owner_split(E, u, l, 2)
        assert len(split[0]) > CE.SEAL_MAX_RECS
    else:
        per_window = CE.SNAP_WINDOW // SC_sealed_len(24 + bsize)
        assert all(len(s) > per_window for s in split)
    page_fn = (lambda q: _small_pages(l[q], bsize)) if small else (lambda q: _random_pages(l[q], bsize, seed=pshift))
    src = _mk(E, pshift, 2, n, tier=True, small=small, max_batch=4096)
    _put(E, src, u, l, page_fn, tier=True)
    plain, sealed = str(tmp_path / "plain"), str(tmp_path / "sealed")
    assert E.save_set([e.h for e in src], plain) == n
    for e in src:
        e.set_file_key(KEY)
    assert E.save_set([e.h for e in src], sealed) == n
    _close(src)
    _ps, pflags, precs = _read_plain(plain)
    raw = open(sealed, "rb").read()
    walked = CE.walk_records(raw)
    assert [(p[3][:16], len(p[3])) for p in precs] == [(struct.pack("<QQ", w[2], w[3]), w[1]) for w in walked]
    if small:
        spshift, sflags, _chain, srecs = SC.read_base(sealed, KEY)
        assert (spshift, sflags) == (pshift, pflags)
        assert srecs == precs
    else:
        # the engine sections are contiguous in the file; windows restart inside each
        owners = [E.owner(_fnv(w[2], w[3]), 2) for w in walked]
        cut = next(k for k in range(1, n) if owners[k] != owners[k - 1])
        assert owners == [owners[0]] * cut + [owners[cut]] * (n - cut)
        bounds = [cut] + [s0 + b for s0, s1 in ((0, cut), (cut, n)) for b in CE.seal_windows([w[1] for w in walked[s0:s1]])]
        assert len(bounds) >= 3
        pick = {k for b in bounds for k in range(b - 2, b + 3) if 0 <= k < n}
        pick |= set(random.Random(pshift).sample(range(n), min(n, 200))) | {0, n - 1}
        got = CE.open_records(raw, KEY, sorted(pick))
        for k in sorted(pick):
            assert got[k] == precs[k], k
    del raw, precs
    a = _mk(E, pshift, 2, n, small=small)
    b = _mk(E, pshift, 2, n, key=KEY, small=small)
    assert E.load_set([e.h for e in a], plain) == n
    assert E.load_set([e.h for e in b], sealed) == n
    assert all(e.load_rejected() == 0 for e in b)
    _same_load(a, b, u, l, bsize)
    _close(a); _close(b)


def SC_sealed_len(n):
    return (n + 48 + 15) & ~15


# ---- D. deltas whose tombstone blocks are long ----

TOMBS = [0, 1, 128, 129, 130, 4096, 100000]


def _check_store(E, engines, model, bsize, all_ids):
    """Every address of all_ids hits with its model page or misses when the model has none."""
    u = np.full(len(all_ids), NH, np.uint64)
    l = np.asarray(all_ids, np.uint64)
    assert sum(e.entries() for e in engines) == len(model)
    got = np.zeros(len(all_ids), bool)
    for e, idx in zip(engines, _owner_split(E, u, l, len(engines))):
        for c0 in range(0, len(idx), 16384):
            q = idx[c0:c0 + 16384]
            out, st = e.get(u[q], l[q])
            hit = st == E.HIT
            assert ((st == E.HIT) | (st == E.MISS)).all()
            want = _small_pages([model.get(int(i), 0) for i in l[q]], bsize)
            assert (out[hit] == want[hit]).all()
            got[q] = hit
    live = np.array([int(i) in model for i in all_ids])
    assert (got == live).all(), np.nonzero(got != live)[0][:10]


def _chain_with_long_tombstone_blocks(E, tmp_path):
    """A sealed chain on two engines: a base of 105 000 pages, then one delta per TOMBS entry with that
    many tombstones, 20 new pages and 5 replaced ones; then delta 8, sealed in Python, with 129
    tombstones and 30 raw pages.  -> (base path, models after each file, every id, engines' nonce)"""
    pshift, bsize = 12, 4096
    n0 = 105000
    ids = np.arange(n0, dtype=np.uint64)
    u = np.full(n0, NH, np.uint64)
    src = _mk(E, pshift, 2, n0 + 1000, key=KEY, small=True)
    _put(E, src, u, ids, lambda q: _small_pages(q, bsize))
    model = {i: i for i in range(n0)}            # id -> page stamp
    base = str(tmp_path / "chain")
    E.snapshot_finish(E.chain_begin([e.h for e in src], base, False))
    models = [dict(model)]
    rng = random.Random(4)
    nxt, stamp = n0, 10 ** 7
    for k, nt in enumerate(TOMBS, 1):
        gone = rng.sample(sorted(model), nt)
        gu = np.full(nt, NH, np.uint64)
        gl = np.array(gone, np.uint64)
        for e, idx in zip(src, _owner_split(E, gu, gl, 2)):
            for c0 in range(0, len(idx), 16384):
                e.unset(gu[idx[c0:c0 + 16384]], gl[idx[c0:c0 + 16384]])
        for i in gone:
            del model[i]
        new = list(range(nxt, nxt + 20)) + rng.sample(sorted(model), 5)
        nxt += 20
        stamps = list(range(stamp, stamp + 25))
        stamp += 25
        nu = np.full(25, NH, np.uint64)
        nl = np.array(new, np.uint64)
        st_of = dict(zip(new, stamps))
        _put(E, src, nu, nl, lambda q: _small_pages([st_of[int(nl[j])] for j in q], bsize),
             ts=np.full(25, 5000 + k, np.uint64))
        model.update(st_of)
        E.snapshot_finish(E.chain_begin([e.h for e in src], base, True))
        models.append(dict(model))
        _cid, kk, tombs, recs = SC.read_delta(f"{base}.d{k}", KEY)
        assert kk == k and sorted(t[1] for t in tombs) == sorted(gone) and all(t[0] == NH for t in tombs)
        assert len(recs) == 25 and all(r is not None for r in recs)
    _close(src)
    # delta 8 from Python: raw-page records (compressed_length 0), no fingerprints
    chain_id = struct.unpack_from("<Q", open(base, "rb").read(), 40)[0]
    gone = rng.sample(sorted(model), 129)
    new = list(range(nxt, nxt + 25)) + rng.sample(sorted(set(model) - set(gone)), 5)
    stamps = list(range(stamp, stamp + 30))
    recs = [(9000 + j, 0, 0, struct.pack("<QQiI", NH, i, 0, 0) + _small_pages([s], bsize)[0].tobytes())
            for j, (i, s) in enumerate(zip(new, stamps))]
    CE.write_delta(f"{base}.d8", KEY, rng.getrandbits(64), pshift, chain_id, 8, [(NH, i) for i in gone], recs)
    for i in gone:
        del model[i]
    model.update(zip(new, stamps))
    models.append(dict(model))
    all_ids = list(range(nxt + 25))
    return base, models, all_ids


def test_long_tombstone_blocks_load_exactly_and_a_flip_ends_the_run(gpu, E, tmp_path):
    base, models, all_ids = _chain_with_long_tombstone_blocks(E, tmp_path)
    nd = len(models) - 1
    _cid, _k, tombs, recs = SC.read_delta(f"{base}.d{nd}", KEY)
    assert len(tombs) == 129 and len(recs) == 30
    for mode in ("chain", "loader"):
        dst = _mk(E, 12, 2, 120000, key=KEY, small=True)
        if mode == "chain":
            assert E.load_chain([e.h for e in dst], base)[1] == nd
        else:
            ld = E.Loader([e.h for e in dst], base)
            while ld.step(9973):
                pass
            assert ld.close()[1] == nd
        assert all(e.load_rejected() == 0 for e in dst)
        _check_store(E, dst, models[nd], 4096, all_ids)
        _close(dst)
    # a flipped tombstone at index 128 or at the last index fails the block's tag: the run ends before it
    for k, nt in enumerate(TOMBS + [129], 1):
        if nt < 129:
            continue
        path = f"{base}.d{k}"
        good = open(path, "rb").read()
        for j in (128, nt - 1):
            open(path, "wb").write(_flip(good, 80 + 16 * j + 9, 0x10))
            with pytest.raises(ValueError):
                SC.read_delta(path, KEY)
            dst = _mk(E, 12, 2, 120000, key=KEY, small=True)
            assert E.load_chain([e.h for e in dst], base)[1] == k - 1, (k, j)
            _check_store(E, dst, models[k - 1], 4096, all_ids)
            _close(dst)
        open(path, "wb").write(good)


# ---- E. files the GPU did not write, and hostile records ----

@pytest.mark.parametrize("pshift,n", [(12, 300), (16, 90), (20, 24)])
@pytest.mark.parametrize("fp", [True, False])
def test_python_sealed_base_loads_as_the_plaintext_save(gpu, E, tmp_path, pshift, n, fp):
    bsize = 1 << pshift
    flags = E.FINGERPRINT if fp else 0
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    src = _mk(E, pshift, 2, n, tier=True, flags=flags)
    _put(E, src, u, l, lambda q: np.stack([E.gen_chunk_host(pshift, int(i), bsize) if i % 3 else
                                           _random_pages([i], bsize)[0] for i in q]), tier=True)
    plain, sealed = str(tmp_path / "plain"), str(tmp_path / "sealed")
    assert E.save_set([e.h for e in src], plain) == n
    _close(src)
    _ps, pflags, precs = _read_plain(plain)
    assert bool(pflags & 1) == fp
    SC.write_base(sealed, KEY, 0x0123456789ABCDEF ^ pshift, pshift, precs, with_fingerprints=fp)
    a = _mk(E, pshift, 2, n, flags=flags)
    b = _mk(E, pshift, 2, n, key=KEY, flags=flags)
    assert E.load_set([e.h for e in a], plain) == n
    assert E.load_set([e.h for e in b], sealed) == n
    assert all(e.load_rejected() == 0 for e in b)
    _same_load(a, b, u, l, bsize, fp=fp)
    _close(a); _close(b)


def _hostile_records(bsize):
    """(records that k_open must refuse for their compressed_length, a raw page it must accept, its page)"""
    page = _random_pages([77], bsize, seed=9)[0]
    bad = [(1, 0, 0, struct.pack("<QQiI", NH, 900001, -1, 0) + page.tobytes()),
           (2, 0, 0, struct.pack("<QQiI", NH, 900002, 100, 0) + bytes(101)),
           (3, 0, 0, struct.pack("<QQiI", NH, 900003, 0, 0) + bytes(100))]
    raw = (4, 0, 0, struct.pack("<QQiI", NH, 900004, 0, 0) + page.tobytes())
    return bad, raw, page


def _mutations(raw: bytes, other: bytes, u0):
    """The sealed file `raw` with records moved: records 3 and 10 swapped, record 20 copied over 30,
    record 40 from `other` (a second sealed save of the same store), u of record 50 and l of record 60
    changed in the clear part.  -> (file, addresses whose record was touched, addresses that now name
    no record)"""
    w = CE.walk_records(raw)
    ow = CE.walk_records(other)
    size = {k: (w[k][1] + 63) & ~15 for k in range(len(w))}
    assert len({w[k][1] for k in (3, 10, 20, 30, 40, 50, 60)}) == 1 and ow[40][2:] == w[40][2:]
    b = bytearray(raw)

    def rec(buf, k, ws):
        return bytes(buf[ws[k][0]:ws[k][0] + size[k]])

    r3, r10, r20 = rec(raw, 3, w), rec(raw, 10, w), rec(raw, 20, w)
    b[w[3][0]:w[3][0] + size[3]] = r10
    b[w[10][0]:w[10][0] + size[10]] = r3
    b[w[30][0]:w[30][0] + size[30]] = r20
    b[w[40][0]:w[40][0] + size[40]] = rec(other, 40, ow)
    struct.pack_into("<Q", b, w[50][0] + 8, w[50][2] ^ 0x100)
    struct.pack_into("<Q", b, w[60][0] + 16, w[60][3] ^ (1 << 40))
    touched = [(w[k][2], w[k][3]) for k in (3, 10, 30, 40, 50, 60)]
    ghosts = [(w[50][2] ^ 0x100, w[50][3]), (w[60][2], w[60][3] ^ (1 << 40))]    # addresses the store has not
    return bytes(b), touched, ghosts


def _addr_arrays(addrs):
    return np.array([a[0] for a in addrs], np.uint64), np.array([a[1] for a in addrs], np.uint64)


def _hostile_file(E, tmp_path):
    """A GPU-written sealed base of 160 raw pages on two engines, with _mutations applied, and a base
    sealed in Python from the same records plus _hostile_records.  -> (paths, u, l, pages, rejected
    addresses, addresses that must miss, raw page address and page)"""
    pshift, bsize, n = 12, 4096, 160
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    pages = _random_pages(range(n), bsize, seed=5)
    src = _mk(E, pshift, 2, n, key=KEY)
    _put(E, src, u, l, lambda q: pages[q])
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    E.save_set([e.h for e in src], a)
    E.save_set([e.h for e in src], b)
    _close(src)
    moved, touched, ghosts = _mutations(open(a, "rb").read(), open(b, "rb").read(), NH)
    bound = str(tmp_path / "bound")
    open(bound, "wb").write(moved)
    _ps, _f, _c, recs = SC.read_base(a, KEY)
    bad, rawrec, page = _hostile_records(bsize)
    lens = str(tmp_path / "lens")
    mixed = recs[:50] + bad[:1] + recs[50:100] + bad[1:] + [rawrec] + recs[100:]
    SC.write_base(lens, KEY, 0xFEEDFACE, pshift, [r for r in mixed], with_fingerprints=True)
    bad_addrs = [struct.unpack_from("<QQ", r[3])[0:2] for r in bad]
    return bound, lens, u, l, pages, touched, ghosts, bad_addrs, (NH, 900004), page


def _assert_rejected_before_any_get(engines, n_loaded, n_rejected, addrs):
    assert sum(e.load_rejected() for e in engines) == n_rejected
    assert sum(e.entries() for e in engines) == n_loaded
    au, al = _addr_arrays(addrs)
    for e in engines:
        assert all(r is None for r in e.read_records(au, al))


def _assert_gets(E, engines, u, l, pages, missing, skip=()):
    miss = set(missing)
    for e, idx in zip(engines, _owner_split(E, u, l, len(engines))):
        out, st = e.get(u[idx], l[idx])
        for j, i in enumerate(idx):
            if (int(u[i]), int(l[i])) in skip:
                continue
            if (int(u[i]), int(l[i])) in miss:
                assert st[j] == E.MISS, i
            else:
                assert st[j] == E.HIT and (out[j] == pages[i]).all(), i


def test_hostile_records_are_rejected_and_the_rest_loads(gpu, E, tmp_path):
    bound, lens, u, l, pages, touched, ghosts, bad_addrs, raw_addr, raw_page = _hostile_file(E, tmp_path)
    n = len(u)
    # authentic tags over a compressed_length k_open must refuse; a raw page is accepted
    dst = _mk(E, 12, 2, n, key=KEY)
    assert E.load_set([e.h for e in dst], lens) == n + 1
    _assert_rejected_before_any_get(dst, n + 1, 3, bad_addrs)
    _assert_gets(E, dst, u, l, pages, [])
    bu, bl = _addr_arrays(bad_addrs + [raw_addr])
    for e, idx in zip(dst, _owner_split(E, bu, bl, 2)):
        out, st = e.get(bu[idx], bl[idx])
        for j, i in enumerate(idx):
            if i < 3:
                assert st[j] == E.MISS
            else:
                assert st[j] == E.HIT and (out[j] == raw_page).all()
    _close(dst)
    # records moved between ordinals or files, or with a changed address: exactly those are rejected
    dst = _mk(E, 12, 2, n, key=KEY)
    assert E.load_set([e.h for e in dst], bound) == n - 6
    _assert_rejected_before_any_get(dst, n - 6, 6, touched + ghosts)
    _assert_gets(E, dst, u, l, pages, touched)
    gu, gl = _addr_arrays(ghosts)
    for e in dst:
        assert (e.get(gu, gl)[1] == E.MISS).all()
    _close(dst)


def test_hostile_records_through_the_loader_while_puts_land(gpu, E, tmp_path):
    bound, lens, u, l, pages, touched, ghosts, bad_addrs, raw_addr, raw_page = _hostile_file(E, tmp_path)
    n = len(u)
    fresh = _random_pages([5000, 5001], 4096, seed=6)
    # (file, records loaded, records rejected, addresses that miss, and two addresses that a rejected
    # record of the file names: one put before the load reads that record, one after the load)
    runs = ((bound, n - 6, 6, touched, touched[3], touched[0]), (lens, n + 1, 3, bad_addrs, bad_addrs[2], bad_addrs[0]))
    for path, n_ok, n_bad, rejected, early, late in runs:
        dst = _mk(E, 12, 2, n, key=KEY)
        ld = E.Loader([e.h for e in dst], path)
        steps = 0
        while True:
            more = ld.step(7)
            steps += 1
            if steps == 1:
                eu, el = _addr_arrays([early])
                dst[E.owner(_fnv(*early), 2)].put(eu, el, fresh[:1])
            if not more:
                break
        lu, ll_ = _addr_arrays([late])
        dst[E.owner(_fnv(*late), 2)].put(lu, ll_, fresh[1:])
        assert ld.close()[0] == n_ok
        assert sum(e.load_rejected() for e in dst) == n_bad
        assert sum(e.entries() for e in dst) == n_ok + 2
        for a, page in ((early, fresh[0]), (late, fresh[1])):
            out, st = dst[E.owner(_fnv(*a), 2)].get(*_addr_arrays([a]))
            assert st[0] == E.HIT and (out[0] == page).all(), (path, a)
        others = [x for x in rejected if x not in (early, late)]
        _assert_gets(E, dst, u, l, pages, others if path == bound else [], skip=(early, late))
        _close(dst)


def test_a_tampered_delta_record_never_serves_the_base_page(gpu, E, tmp_path):
    pshift, bsize, n = 12, 4096, 200
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    pages = _random_pages(range(n), bsize, seed=7)
    src = _mk(E, pshift, 2, n, key=KEY)
    _put(E, src, u, l, lambda q: pages[q])
    base = str(tmp_path / "chain")
    E.snapshot_finish(E.chain_begin([e.h for e in src], base, False))
    upd = np.arange(40, 60)
    new_pages = _random_pages(upd, bsize, seed=8)
    _put(E, src, u[upd], l[upd], lambda q: new_pages[q], ts=np.full(len(upd), 7777, np.uint64))
    E.snapshot_finish(E.chain_begin([e.h for e in src], base, True))
    _close(src)
    raw = open(base + ".d1", "rb").read()
    w = CE.walk_records(raw)
    victim = 7
    a = w[victim][2:]
    open(base + ".d1", "wb").write(_flip(raw, w[victim][0] + 24 + 100, 0x08))
    want = pages.copy()
    want[upd] = new_pages
    for mode in ("chain", "loader"):
        dst = _mk(E, pshift, 2, n, key=KEY)
        if mode == "chain":
            assert E.load_chain([e.h for e in dst], base) == (n - 1, 1)
        else:
            ld = E.Loader([e.h for e in dst], base)
            while ld.step(13):
                pass
            assert ld.close() == (n - 1, 1)
        _assert_rejected_before_any_get(dst, n - 1, 1, [a])
        _assert_gets(E, dst, u, l, want, [a])
        _close(dst)


# ---- F. loads into engines that stage one record at a time ----

@pytest.mark.parametrize("pshift", [12, 16])
def test_every_max_batch_loads_what_the_store_saved(gpu, E, tmp_path, pshift):
    bsize, n = 1 << pshift, 40
    u = np.full(n, NH, np.uint64)
    l = np.arange(n, dtype=np.uint64)
    pages = _random_pages(range(n), bsize, seed=pshift)
    src = _mk(E, pshift, 2, n)
    _put(E, src, u, l, lambda q: pages[q])
    plain, sealed = str(tmp_path / "plain"), str(tmp_path / "sealed")
    assert E.save_set([e.h for e in src], plain) == n
    for e in src:
        e.set_file_key(KEY)
    assert E.save_set([e.h for e in src], sealed) == n
    _close(src)
    assert all(len(r[3]) >= 24 + bsize for r in _read_plain(plain)[2])      # incompressible: the largest records
    ref = _mk(E, pshift, 2, n)
    assert E.load_set([e.h for e in ref], plain) == n
    for mb in (1, 2, 256):
        for path, key in ((plain, None), (sealed, KEY)):
            for mode in ("set", "loader") if mb == 1 else ("set",):
                dst = _mk(E, pshift, 2, n, key=key, max_batch=mb)
                if mode == "set":
                    assert E.load_set([e.h for e in dst], path) == n, (mb, path)
                else:
                    ld = E.Loader([e.h for e in dst], path)
                    while ld.step(3):
                        pass
                    assert ld.close()[0] == n
                _same_load(ref, dst, u, l, bsize, samples=1024, what=(mb, key is None, mode))
                _assert_gets(E, dst, u, l, pages, [])
                _close(dst)
    _close(ref)
