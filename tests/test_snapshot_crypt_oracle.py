"""Pins tests/snapshot_crypt.py, the pure-Python ChaCha20-Poly1305 the sealed-file tests check the GPU
against, to RFC 8439's vectors and to record-sized cases sealed by the `cryptography` package
(tests/golden/chacha20poly1305.json, made by tools/gen_crypt_golden.py), and to `cryptography` itself
where that package imports."""
import hashlib
import json
import os
import random
import struct

import pytest

import snapshot_crypt as SC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "chacha20poly1305.json")
H = bytes.fromhex


@pytest.fixture(scope="module")
def vectors():
    with open(GOLDEN) as f:
        return json.load(f)


def record_message(case) -> bytes:
    return b"\xff" * case["len"] if case["ff"] else random.Random(case["seed"]).randbytes(case["len"])


def test_chacha20_rfc(vectors):
    for v in vectors["chacha20"]:
        assert SC.chacha20(H(v["key"]), v["counter"], H(v["nonce"]), H(v["plaintext"])) == H(v["ciphertext"])


def test_poly1305_rfc_and_edge_cases(vectors):
    assert len(vectors["poly1305"]) >= 7
    for v in vectors["poly1305"]:
        assert SC.poly1305(H(v["key"]), H(v["msg"])) == H(v["tag"]), v["name"]


def test_poly1305_key_generation_rfc(vectors):
    for v in vectors["keygen"]:
        assert SC.poly1305_key_gen(H(v["key"]), H(v["nonce"])) == H(v["poly_key"])


def test_aead_rfc(vectors):
    for v in vectors["aead"]:
        sealed = SC.seal(H(v["key"]), H(v["nonce"]), H(v["aad"]), H(v["plaintext"]))
        assert sealed == H(v["sealed"])
        assert SC.open_(H(v["key"]), H(v["nonce"]), H(v["aad"]), sealed) == H(v["plaintext"])


@pytest.mark.parametrize("limit", [65, 24 + 4096])
def test_aead_record_sizes(vectors, limit):
    """The stored cases whole; hashed ones up to 4 KiB here (the GPU tests run every size)."""
    for v in vectors["records"]:
        if v["len"] > limit or ("sha256" in v) != (limit > 65):
            continue
        m = record_message(v)
        sealed = SC.seal(H(v["key"]), H(v["nonce"]), H(v["aad"]), m)
        if "sealed" in v:
            assert sealed == H(v["sealed"])
        else:
            assert hashlib.sha256(sealed).hexdigest() == v["sha256"]


def test_open_rejects_each_flipped_part():
    key, nonce, aad, m = bytes(range(32)), bytes(12), b"A" * 24, bytes(range(100))
    sealed = SC.seal(key, nonce, aad, m)
    for at in (0, 50, 99, 100, 115):
        bad = bytearray(sealed)
        bad[at] ^= 1
        assert SC.open_(key, nonce, aad, bytes(bad)) is None
    assert SC.open_(key, nonce, b"B" + aad[1:], sealed) is None
    assert SC.open_(key, nonce, aad, sealed) == m


def test_sealed_base_round_trip(tmp_path):
    key = bytes(range(1, 33))
    recs = [(7 + i, i, 2 * i, struct.pack("<QQiI", 5, i, 0, 0) + bytes([i]) * 64) for i in range(5)]
    p = str(tmp_path / "snap")
    SC.write_base(p, key, 0x1234, 12, recs, chain_id=9)
    pshift, _flags, chain, out = SC.read_base(p, key)
    assert pshift == 12 and chain == 9 and out == recs
    with pytest.raises(ValueError):
        SC.read_base(p, bytes(32))
    raw = open(p, "rb").read()
    assert raw[:8] == b"CMB200E1" and len(raw) == 80 + 5 * ((88 + 48 + 15) & ~15)


def test_against_cryptography():
    aead = pytest.importorskip("cryptography.hazmat.primitives.ciphers.aead")
    rng = random.Random(3)
    for n in (0, 1, 15, 16, 17, 63, 64, 65, 200, 1000):
        key, nonce, aad, m = rng.randbytes(32), rng.randbytes(12), rng.randbytes(rng.randrange(40)), rng.randbytes(n)
        assert SC.seal(key, nonce, aad, m) == aead.ChaCha20Poly1305(key).encrypt(nonce, m, aad)
