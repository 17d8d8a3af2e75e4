"""CPU checks of tests/crypt_edges.py, the helpers tests/test_gpu_crypt_edges.py drives the GPU's
ChaCha20-Poly1305 with: every Poly1305 target is reached (under tests/snapshot_crypt.py and, where it
imports, the `cryptography` package), the nonce search returns what it claims, and the sealed-delta
writer and the record walker round-trip through snapshot_crypt's reader."""
import random
import struct

import pytest

import crypt_edges as CE
import snapshot_crypt as SC

KEY = bytes(range(0x40, 0x60))


def _targets():
    for name, t in [(str(t), t) for t in CE.SMALL_TARGETS] + CE.EDGE_TARGETS:
        for prefix in CE.TARGET_PREFIXES:
            for aad_len in CE.TARGET_AADS:
                yield name, t, prefix, aad_len


def test_target_message_reaches_every_target():
    rng = random.Random(21)
    try:
        from cryptography.hazmat.primitives.ciphers.aead import ChaCha20Poly1305
    except ImportError:
        ChaCha20Poly1305 = None
    for name, t, prefix, aad_len in _targets():
        aad = rng.randbytes(aad_len)
        nonce, pt, ct, T = CE.find_target(KEY, aad, prefix, t, rng)
        r, s = CE.poly_rs(KEY, nonce)
        mac = CE.mac_input(aad, ct)
        assert len(ct) == prefix + 16 and 0 <= T < CE.P
        assert CE.residue(r, mac) == T, name
        # snapshot_crypt's Poly1305 with s = 0 gives the residue mod 2^128, with the real s the tag
        assert SC.poly1305(r.to_bytes(16, "little") + bytes(16), mac) == (T & CE.M128).to_bytes(16, "little")
        tag = ((T + s) & CE.M128).to_bytes(16, "little")
        assert SC.seal(KEY, nonce, aad, pt) == ct + tag, name
        if name == "tag 0":
            assert tag == bytes(16)
        if name == "tag 1":
            assert tag == b"\x01" + bytes(15)
        if ChaCha20Poly1305 is not None:
            assert ChaCha20Poly1305(KEY).encrypt(nonce, pt, aad) == ct + tag, name


def test_targets_name_the_edges_they_claim():
    double = dict((n, t) for n, t in CE.EDGE_TARGETS)["double carry"]
    limbs = CE.limbs26(double)
    assert limbs[1] == (1 << 26) - 1 and limbs[0] >= (1 << 26) - 5
    assert CE.limbs26((1 << 104) - 1)[:4] == [(1 << 26) - 1] * 4
    assert all(t + CE.P < 1 << 130 for t in CE.SMALL_TARGETS)


def test_target_message_without_a_prefix_is_one_draw():
    rng = random.Random(5)
    got = [CE.target_message(KEY, rng.randbytes(12), b"", 0, 3) for _ in range(64)]
    # m < 2^128 for about one residue in four
    assert 4 <= sum(g is not None for g in got) <= 40


def test_best_r_nonce_is_the_best_of_those_tried():
    tries = 4096
    nonce, bits = CE.best_r_nonce(KEY, tries=tries, seed=3)
    r, _s = CE.poly_rs(KEY, nonce)
    assert bin(r).count("1") == bits
    # the numpy ChaCha20 block 0 against snapshot_crypt's, on a sample of the nonces tried
    rng = random.Random(2)
    for i in rng.sample(range(tries), 64):
        n = struct.pack("<III", 3, i, 0)
        assert bin(CE.poly_rs(KEY, n)[0]).count("1") <= bits
    clamp_bits = bin(CE.R_CLAMP).count("1")
    # a random r has about half its 106 free bits set; the best of 4096 is well above that
    assert clamp_bits // 2 + 10 <= bits <= clamp_bits


def _record(u, l, payload, clen=None):
    return struct.pack("<QQiI", u, l, len(payload) if clen is None else clen, 0) + payload


@pytest.mark.parametrize("nt", [0, 1, 128, 129, 4096])
def test_write_delta_round_trips_through_snapshot_crypt(tmp_path, nt):
    rng = random.Random(nt)
    tombs = [(7, rng.randrange(1 << 40)) for _ in range(nt)]
    recs = [(100 + i, i, 3 * i, _record(7, 1000 + i, rng.randbytes(rng.randrange(1, 300)))) for i in range(9)]
    p = str(tmp_path / "d")
    CE.write_delta(p, KEY, 0xABCDEF, 12, 77, 3, tombs, recs, with_fingerprints=True)
    chain, k, got_t, got_r = SC.read_delta(p, KEY)
    assert (chain, k, got_t, got_r) == (77, 3, tombs, recs)
    raw = open(p, "rb").read()
    assert raw[:8] == b"CMB200F1" and struct.unpack_from("<Q", raw, 56)[0] == 0xABCDEF
    assert [(u, l) for _p, _n, u, l in CE.walk_records(raw)] == [CE.walk_records(raw)[i][2:] for i in range(9)]
    assert CE.open_records(raw, KEY, [0, 8]) == {0: recs[0], 8: recs[8]}
    if nt:
        # a flipped tombstone fails the tombstone tag
        bad = bytearray(raw)
        bad[80 + 16 * (nt - 1) + 3] ^= 1
        open(p, "wb").write(bytes(bad))
        with pytest.raises(ValueError):
            SC.read_delta(p, KEY)


def test_walk_and_open_records_of_a_base(tmp_path):
    rng = random.Random(9)
    recs = [(i, 0, 0, _record(5, i, rng.randbytes(rng.randrange(1, 200)))) for i in range(20)]
    p = str(tmp_path / "b")
    SC.write_base(p, KEY, 42, 12, recs)
    raw = open(p, "rb").read()
    walked = CE.walk_records(raw)
    assert [(n, u, l) for _p, n, u, l in walked] == [(len(r[3]), 5, i) for i, r in enumerate(recs)]
    assert CE.open_records(raw, KEY, range(20)) == dict(enumerate(recs))
    # record 4's bytes in the place of record 3 (its nonce is 2 + 4, not 2 + 3) do not open there
    a, b = walked[3], walked[4]
    swapped = raw[:a[0]] + raw[b[0]:] + raw[a[0]:b[0]]
    swapped = swapped[:a[0] + ((b[1] + 63) & ~15)] + raw[a[0]:b[0]] + raw[b[0] + ((b[1] + 63) & ~15):]
    got = CE.open_records(swapped, KEY, [3, 4])
    assert got == {3: None, 4: None}


def test_records_with_a_bad_length_keep_an_authentic_tag(tmp_path):
    """The hostile records of the GPU test: an authentic tag over a compressed_length that the load must
    refuse.  snapshot_crypt opens them; only the engine's length check may reject them."""
    bsize = 4096
    recs = [(1, 0, 0, _record(9, 0, bytes(bsize), clen=-1)),
            (2, 0, 0, _record(9, 1, bytes(101), clen=100)),
            (3, 0, 0, _record(9, 2, bytes(100), clen=0)),
            (4, 0, 0, _record(9, 3, bytes(bsize), clen=0))]
    p = str(tmp_path / "b")
    SC.write_base(p, KEY, 1, 12, recs)
    assert SC.read_base(p, KEY)[3] == recs


def test_seal_windows():
    assert CE.seal_windows([24 + 4096] * 10) == []
    assert CE.seal_windows([40] * (3 * CE.SEAL_MAX_RECS + 5)) == [CE.SEAL_MAX_RECS * j for j in (1, 2, 3)]
    big = 24 + (1 << 16)
    per = CE.SNAP_WINDOW // ((big + 63) & ~15)
    assert CE.seal_windows([big] * (2 * per + 1)) == [per, 2 * per]
