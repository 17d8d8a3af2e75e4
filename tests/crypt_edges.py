"""TEST INFRASTRUCTURE ONLY — helpers that drive the sealed-file tests to their edges, on top of
tests/snapshot_crypt.py (SC):

    target_message   a ciphertext whose Poly1305 residue, before + s, is a chosen value T
    best_r_nonce     a nonce whose clamped Poly1305 r has the most bits set among many tried
    write_delta      a sealed delta ("CMB200F1"), restated from DESIGN.md §2, so that a test can hand
                     the engine a delta it did not write
    walk_records     the offsets and clear parts of a sealed base's or delta's records, and
                     open_records, which opens only chosen ones (a large file decrypts in part)
    seal_windows     the ordinals at which the engine's sealed writer starts a new window
"""
from __future__ import annotations

import random
import struct

import numpy as np

import snapshot_crypt as SC

P = SC.P1305
M128 = (1 << 128) - 1
R_CLAMP = 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF
SNAP_WINDOW = 64 << 20          # sealed bytes per window of the engine's writer
SEAL_MAX_RECS = 1 << 16         # records per window


def poly_rs(key: bytes, nonce: bytes):
    """(r clamped, s) of the one-time Poly1305 key of (key, nonce)."""
    pk = SC.poly1305_key_gen(key, nonce)
    return int.from_bytes(pk[:16], "little") & R_CLAMP, int.from_bytes(pk[16:], "little")


def mac_input(aad: bytes, ct: bytes) -> bytes:
    """What RFC 8439 §2.8 feeds to Poly1305."""
    return aad + SC._pad16(aad) + ct + SC._pad16(ct) + struct.pack("<QQ", len(aad), len(ct))


def residue(r: int, msg: bytes) -> int:
    """The Poly1305 accumulator of msg mod 2^130 - 5, before + s."""
    acc = 0
    for i in range(0, len(msg), 16):
        acc = (acc + int.from_bytes(msg[i:i + 16] + b"\x01", "little")) * r % P
    return acc


def target_message(key: bytes, nonce: bytes, aad: bytes, prefix_len: int, T: int, rng=None, tries: int = 64):
    """(plaintext, ciphertext) of prefix_len + 16 bytes whose AEAD tag residue, before + s, is T (< p),
    or None when `tries` draws of the random prefix found none (with no prefix there is one draw).

    The last ciphertext block m is a full block, followed by the lengths block, so its coefficient is
    r^2: h(m) = h(0) + m r^2 mod p, and m = (T - h(0)) r^-2 mod p, taken when it is below 2^128."""
    assert prefix_len % 16 == 0 and 0 <= T < P
    rng = rng or random.Random(0)
    r, _s = poly_rs(key, nonce)
    inv_r2 = pow(r * r % P, -1, P)
    for _ in range(tries if prefix_len else 1):
        prefix = rng.randbytes(prefix_len)
        h0 = residue(r, mac_input(aad, prefix + bytes(16)))
        m = (T - h0) * inv_r2 % P
        if m <= M128:
            ct = prefix + m.to_bytes(16, "little")
            return SC.chacha20(key, 1, nonce, ct), ct
    return None


def find_target(key: bytes, aad: bytes, prefix_len: int, target, rng):
    """(nonce, plaintext, ciphertext, T): target_message under the first random nonce that reaches
    target(s) (an int, or a function of the one-time key's s)."""
    while True:
        nonce = rng.randbytes(12)
        _r, s = poly_rs(key, nonce)
        T = target(s) if callable(target) else target
        got = target_message(key, nonce, aad, prefix_len, T, rng)
        if got is not None:
            return nonce, got[0], got[1], T


def limbs26(x: int):
    return [(x >> (26 * i)) & 0x3FFFFFF for i in range(5)]


# Residues that reach the edges of the final reduction: h >= p or not, the carry out of limb 1, the
# 2^128 and 2^129 bits, and the + s mod 2^128 carry through all four words (tag 0 and 1).
SMALL_TARGETS = [0, 1, 2, 3, 4]        # each has two representatives below 2^130: T and T + p
EDGE_TARGETS = [
    ("p-1", P - 1), ("p-2", P - 2),
    ("2^128-1", M128), ("2^128", 1 << 128), ("2^129", 1 << 129),
    ("2^104-1", (1 << 104) - 1),
    ("double carry", ((1 << 26) - 1) << 26 | ((1 << 26) - 3)),
    ("tag 0", lambda s: (-s) & M128), ("tag 1", lambda s: ((-s) & M128) + 1),
]
# the last block in lane 0, in lane 31, and in lane 0's second group; the AAD empty, short, and longer
# than a warp's first round of groups
TARGET_PREFIXES = [0, 1984, 2048]
TARGET_AADS = [0, 24, 2064]


def best_r_nonce(key: bytes, tries: int = 1 << 17, seed: int = 1):
    """(nonce, popcount of r): among `tries` nonces {seed's counter, i}, the one whose clamped r has the
    most bits set (ChaCha20 block 0 of every nonce at once, as numpy columns)."""
    i = np.arange(tries, dtype=np.uint64)
    s = np.zeros((16, tries), np.uint32)
    s[0:4] = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], np.uint32)[:, None]
    s[4:12] = np.frombuffer(key, "<u4")[:, None]
    s[13] = np.uint32(seed)
    s[14] = (i & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    s[15] = (i >> np.uint64(32)).astype(np.uint32)
    x = s.copy()

    def rotl(v, n):
        return (v << np.uint32(n)) | (v >> np.uint32(32 - n))

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    w = (x[0:4] + s[0:4]) & np.array([0x0FFFFFFF, 0x0FFFFFFC, 0x0FFFFFFC, 0x0FFFFFFC], np.uint32)[:, None]
    bits = np.unpackbits(w.T.copy().view(np.uint8), axis=1).sum(axis=1)
    best = int(np.argmax(bits))
    return struct.pack("<III", seed, best & 0xFFFFFFFF, best >> 32), int(bits[best])


# ---- sealed files ----
def write_delta(path: str, key: bytes, nonce64: int, pshift: int, chain_id: int, k: int, tombstones, records,
                with_fingerprints: bool = False) -> None:
    """A sealed delta: tests/snapshot_chain.py's 64-byte header under "CMB200F1" with the file nonce in its
    last 8 bytes, the tag of seal(i = 0, AAD = header, ""), the clear tombstones {u64 u, u64 l}, the tag
    of seal(i = 1, AAD = tombstones, ""), then the records sealed as in a base (i = 2 + ordinal).
    tombstones: [(u, l)]; records: [(ts, fp_hi, fp_lo, record)]."""
    tombstones, records = list(tombstones), list(records)
    h = SC.DELTA_MAGIC + struct.pack("<IIQIIQQQQ", 1, pshift, chain_id, k, 1 if with_fingerprints else 0,
                                     len(tombstones), len(records), sum(len(r[3]) for r in records), nonce64)
    tb = b"".join(struct.pack("<QQ", u, l) for u, l in tombstones)
    with open(path, "wb") as f:
        f.write(h)
        f.write(SC.seal(key, SC.file_nonce(nonce64, 0), h, b""))
        f.write(tb)
        f.write(SC.seal(key, SC.file_nonce(nonce64, 1), tb, b""))
        for j, (ts, hi, lo, rec) in enumerate(records):
            f.write(SC.seal_record(key, nonce64, j, ts, hi, lo, rec))


def file_layout(raw: bytes):
    """(nonce64, offset of the first record, record count) of a sealed base or delta."""
    if raw[:8] == SC.BASE_MAGIC:
        (count,) = struct.unpack_from("<Q", raw, 16)
        (nonce64,) = struct.unpack_from("<Q", raw, 48)
        return nonce64, 80, count
    assert raw[:8] == SC.DELTA_MAGIC, "not a sealed file"
    nt, nr = struct.unpack_from("<QQ", raw, 32)
    (nonce64,) = struct.unpack_from("<Q", raw, 56)
    return nonce64, 80 + 16 * nt + 16, nr


def walk_records(raw: bytes):
    """[(offset, len, u, l)] of every record of a sealed base or delta, from the clear parts alone."""
    _n64, pos, count = file_layout(raw)
    out = []
    for _ in range(count):
        n, zero, u, l = struct.unpack_from("<IIQQ", raw, pos)
        assert zero == 0
        out.append((pos, n, u, l))
        pos += (n + 48 + 15) & ~15
    assert pos == len(raw)
    return out


def open_records(raw: bytes, key: bytes, ordinals):
    """{ordinal: (ts, fp_hi, fp_lo, record) or None} for the chosen records of a sealed base or delta."""
    nonce64 = file_layout(raw)[0]
    recs = walk_records(raw)
    out = {}
    for k in ordinals:
        pos, n, _u, _l = recs[k]
        clear = raw[pos:pos + 24]
        pt = SC.open_(key, SC.file_nonce(nonce64, 2 + k), clear, raw[pos + 24:pos + 24 + n + 8 + 16])
        out[k] = None if pt is None else (*struct.unpack("<QQQ", pt[:24]), clear[8:24] + pt[24:])
    return out


def seal_windows(lens):
    """The ordinals (> 0) of one engine section whose record starts a new window of the sealed writer,
    given the section's record lengths in file order: a window ends before 64 MiB of sealed bytes or at
    65 536 records."""
    starts, nbytes, nrec = [], 0, 0
    for k, n in enumerate(lens):
        sb = (n + 48 + 15) & ~15
        if nrec == SEAL_MAX_RECS or nbytes + sb > SNAP_WINDOW:
            starts.append(k)
            nbytes, nrec = 0, 0
        nbytes += sb
        nrec += 1
    return starts
