"""TEST INFRASTRUCTURE ONLY — a pure-Python ChaCha20-Poly1305 (RFC 8439 §2.8) and an independent reader /
writer of sealed snapshot files, restated from include/cachemap_b200.h and DESIGN.md §2 "Encryption at
rest", so that the tests can check the files the engine writes and hand it files it did not write.

    sealed base   "CMB200E1": oracle/snapshot.py's 64-byte header (chain id at bytes 40..47) with the
                  64-bit file nonce at bytes 48..55, then the 16-byte tag of seal(i = 0, AAD = header, "")
    sealed delta  "CMB200F1": tests/snapshot_chain.py's 64-byte delta header with the file nonce in its
                  last 8 bytes, then the tag of seal(i = 0, AAD = header, ""), the clear 16-byte
                  tombstones, and the tag of seal(i = 1, AAD = tombstones, "")
    record        {u32 len, u32 0, u64 u, u64 l}  (AAD)
                  ciphertext of {u64 ts, u64 fp_hi, u64 fp_lo, the record's len - 16 bytes after {u, l}}
                  16-byte tag, zeros to a multiple of 16
    nonce         {u64 file nonce, u32 i} little-endian; i = 2 + the record's ordinal in the file
"""
from __future__ import annotations

import struct

import numpy as np

BASE_MAGIC = b"CMB200E1"
DELTA_MAGIC = b"CMB200F1"
M32 = 0xFFFFFFFF
P1305 = (1 << 130) - 5


# ---- ChaCha20 (§2.3, §2.4) ----
def _qr(x, a, b, c, d):
    x[a] = (x[a] + x[b]) & M32; x[d] ^= x[a]; x[d] = ((x[d] << 16) | (x[d] >> 16)) & M32
    x[c] = (x[c] + x[d]) & M32; x[b] ^= x[c]; x[b] = ((x[b] << 12) | (x[b] >> 20)) & M32
    x[a] = (x[a] + x[b]) & M32; x[d] ^= x[a]; x[d] = ((x[d] << 8) | (x[d] >> 24)) & M32
    x[c] = (x[c] + x[d]) & M32; x[b] ^= x[c]; x[b] = ((x[b] << 7) | (x[b] >> 25)) & M32


def chacha20_block(key: bytes, counter: int, nonce: bytes) -> bytes:
    s = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574, *struct.unpack("<8I", key), counter & M32,
         *struct.unpack("<3I", nonce)]
    x = list(s)
    for _ in range(10):
        _qr(x, 0, 4, 8, 12); _qr(x, 1, 5, 9, 13); _qr(x, 2, 6, 10, 14); _qr(x, 3, 7, 11, 15)
        _qr(x, 0, 5, 10, 15); _qr(x, 1, 6, 11, 12); _qr(x, 2, 7, 8, 13); _qr(x, 3, 4, 9, 14)
    return struct.pack("<16I", *[(a + b) & M32 for a, b in zip(x, s)])


def chacha20(key: bytes, counter: int, nonce: bytes, data: bytes) -> bytes:
    """The keystream from block `counter` on, xored into data: chacha20_block's rounds on every block at
    once, as numpy uint32 columns."""
    nb = (len(data) + 63) // 64
    if nb == 0:
        return b""
    s = np.zeros((16, nb), np.uint32)
    s[0:4] = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], np.uint32)[:, None]
    s[4:12] = np.frombuffer(key, "<u4")[:, None]
    s[12] = (np.arange(nb, dtype=np.uint64) + counter).astype(np.uint32)
    s[13:16] = np.frombuffer(nonce, "<u4")[:, None]
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
    ks = (x + s).T.astype("<u4").tobytes()[:len(data)]
    return (np.frombuffer(data, np.uint8) ^ np.frombuffer(ks, np.uint8)).tobytes()


# ---- Poly1305 (§2.5) ----
def poly1305(key: bytes, msg: bytes) -> bytes:
    r = int.from_bytes(key[:16], "little") & 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF
    s = int.from_bytes(key[16:32], "little")
    acc = 0
    for i in range(0, len(msg), 16):
        n = int.from_bytes(msg[i:i + 16] + b"\x01", "little")
        acc = (acc + n) * r % P1305
    return ((acc + s) & ((1 << 128) - 1)).to_bytes(16, "little")


def poly1305_key_gen(key: bytes, nonce: bytes) -> bytes:
    return chacha20_block(key, 0, nonce)[:32]


def _pad16(b: bytes) -> bytes:
    return b"\0" * ((16 - len(b) % 16) % 16)


# ---- AEAD (§2.8) ----
def seal(key: bytes, nonce: bytes, aad: bytes, plaintext: bytes) -> bytes:
    """ciphertext || tag"""
    ct = chacha20(key, 1, nonce, plaintext)
    mac = aad + _pad16(aad) + ct + _pad16(ct) + struct.pack("<QQ", len(aad), len(ct))
    return ct + poly1305(poly1305_key_gen(key, nonce), mac)


def open_(key: bytes, nonce: bytes, aad: bytes, sealed: bytes):
    """plaintext, or None when the tag is wrong"""
    ct, tag = sealed[:-16], sealed[-16:]
    mac = aad + _pad16(aad) + ct + _pad16(ct) + struct.pack("<QQ", len(aad), len(ct))
    if poly1305(poly1305_key_gen(key, nonce), mac) != tag:
        return None
    return chacha20(key, 1, nonce, ct)


def file_nonce(nonce64: int, i: int) -> bytes:
    return struct.pack("<QI", nonce64, i)


# ---- sealed files ----
def seal_record(key: bytes, nonce64: int, ordinal: int, ts: int, fp_hi: int, fp_lo: int, rec: bytes) -> bytes:
    clear = struct.pack("<II", len(rec), 0) + rec[:16]
    body = seal(key, file_nonce(nonce64, 2 + ordinal), clear, struct.pack("<QQQ", ts, fp_hi, fp_lo) + rec[16:])
    out = clear + body
    return out + b"\0" * ((16 - len(out) % 16) % 16)


def _read_sealed_records(f, key: bytes, nonce64: int, count: int):
    """[(ts, fp_hi, fp_lo, record) or None for a record that does not open]"""
    out = []
    for k in range(count):
        clear = f.read(24)
        if len(clear) != 24:
            raise ValueError("truncated record")
        n, zero = struct.unpack("<II", clear[:8])
        if zero:
            raise ValueError("corrupt record")
        total = (n + 48 + 15) & ~15
        rest = f.read(total - 24)
        if len(rest) != total - 24:
            raise ValueError("truncated record")
        pt = open_(key, file_nonce(nonce64, 2 + k), clear, rest[:n + 8 + 16])
        if pt is None:
            out.append(None)
            continue
        ts, hi, lo = struct.unpack("<QQQ", pt[:24])
        out.append((ts, hi, lo, clear[8:24] + pt[24:]))
    return out


def read_base(path: str, key: bytes):
    """(pshift, flags, chain id, [(ts, fp_hi, fp_lo, record) or None]) of a sealed base."""
    with open(path, "rb") as f:
        h = f.read(64)
        if h[:8] != BASE_MAGIC:
            raise ValueError("not a sealed snapshot")
        _v, pshift, records, _bytes, flags = struct.unpack("<IIQQI", h[8:36])
        (chain_id,) = struct.unpack_from("<Q", h, 40)
        (nonce64,) = struct.unpack_from("<Q", h, 48)
        tag = f.read(16)
        if open_(key, file_nonce(nonce64, 0), h, tag) is None:
            raise ValueError("header does not open with this key")
        return pshift, flags, chain_id, _read_sealed_records(f, key, nonce64, records)


def write_base(path: str, key: bytes, nonce64: int, pshift: int, records, chain_id: int = 0,
               with_fingerprints: bool = False) -> None:
    """records: [(ts, fp_hi, fp_lo, record)]"""
    h = bytearray(64)
    h[:8] = BASE_MAGIC
    struct.pack_into("<IIQQI", h, 8, 1, pshift, len(records), sum(len(r[3]) for r in records),
                     1 if with_fingerprints else 0)
    struct.pack_into("<Q", h, 40, chain_id)
    struct.pack_into("<Q", h, 48, nonce64)
    with open(path, "wb") as f:
        f.write(bytes(h))
        f.write(seal(key, file_nonce(nonce64, 0), bytes(h), b""))
        for k, (ts, hi, lo, rec) in enumerate(records):
            f.write(seal_record(key, nonce64, k, ts, hi, lo, rec))


def read_delta(path: str, key: bytes):
    """(chain id, k, [tombstone (u, l)], [(ts, fp_hi, fp_lo, record) or None]) of a sealed delta."""
    with open(path, "rb") as f:
        h = f.read(64)
        if h[:8] != DELTA_MAGIC:
            raise ValueError("not a sealed delta")
        _v, _pshift, chain_id, k, _flags, nt, nr, _nb, nonce64 = struct.unpack("<IIQIIQQQQ", h[8:64])
        if open_(key, file_nonce(nonce64, 0), h, f.read(16)) is None:
            raise ValueError("delta header does not open with this key")
        tb = f.read(16 * nt)
        if open_(key, file_nonce(nonce64, 1), tb, f.read(16)) is None:
            raise ValueError("tombstones do not open with this key")
        tombs = [struct.unpack_from("<QQ", tb, 16 * j) for j in range(nt)]
        return chain_id, k, tombs, _read_sealed_records(f, key, nonce64, nr)
