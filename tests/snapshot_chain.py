"""TEST INFRASTRUCTURE ONLY — independent writer / reader of snapshot chains (cmb200_chain_begin /
cmb200_load_chain), next to oracle/snapshot.py's base format, restated from include/cachemap_b200.h and
DESIGN.md §2 so that the tests can check the files the engine writes and hand it files it did not write.

    base        oracle/snapshot.py's file, with the 64-bit chain id in header bytes 40..47 (0: no chain)
    delta k     <base>.d<k>:
      header    "CMB200D1" | u32 version = 1 | u32 pshift | u64 chain id | u32 k | u32 flags |
                u64 tombstones | u64 records | u64 record bytes | pad to 64
      tombstones  16-byte addresses {u64 u, u64 l}: live at tick k-1, not live at tick k
      records   as in the base: u64 ts | u64 fp_hi | u64 fp_lo | u32 len | u32 0 | len bytes | pad to 16

The store a chain describes is the base, then for each delta in order its tombstones removed and its
records put.  A chain's valid run is the base plus deltas 1, 2, ... while each is present, whole, of the
base's chain id and numbered in sequence; the first that is not ends the run, and nothing after it counts.
"""
from __future__ import annotations

import os
import struct

from oracle import snapshot

DELTA_MAGIC = b"CMB200D1"


def addr_of(record_bytes: bytes):
    """(u, l) of a record: the first 16 bytes of its 24-byte prefix."""
    return struct.unpack("<QQ", record_bytes[:16])


def _write_records(f, records) -> None:
    for ts, hi, lo, rec in records:
        f.write(struct.pack("<QQQII", ts, hi, lo, len(rec), 0))
        f.write(rec)
        f.write(b"\0" * ((16 - len(rec) % 16) % 16))


def _read_records(f, count):
    out = []
    for _ in range(count):
        head = f.read(32)
        if len(head) != 32:
            raise ValueError("truncated record header")
        ts, hi, lo, n, _zero = struct.unpack("<QQQII", head)
        rec = f.read(n)
        pad = f.read((16 - n % 16) % 16)
        if len(rec) != n or len(pad) != (16 - n % 16) % 16:
            raise ValueError("truncated record")
        out.append((ts, hi, lo, rec))
    return out


def write_base(path: str, pshift: int, records, chain_id: int, with_fingerprints: bool = False) -> None:
    snapshot.write_snapshot(path, pshift, records, with_fingerprints)
    with open(path, "r+b") as f:
        f.seek(40)
        f.write(struct.pack("<Q", chain_id))


def read_chain_id(path: str) -> int:
    with open(path, "rb") as f:
        head = f.read(64)
    assert head[:8] == snapshot.MAGIC, "not a snapshot"
    return struct.unpack("<Q", head[40:48])[0]


def write_delta(path: str, pshift: int, chain_id: int, k: int, tombstones, records,
                with_fingerprints: bool = False) -> None:
    """tombstones: iterable of (u, l); records: iterable of (ts, fp_hi, fp_lo, record_bytes)."""
    tombstones, records = list(tombstones), list(records)
    total = sum(len(r[3]) for r in records)
    with open(path, "wb") as f:
        f.write(DELTA_MAGIC + struct.pack("<IIQIIQQQ", 1, pshift, chain_id, k, 1 if with_fingerprints else 0,
                                          len(tombstones), len(records), total) + b"\0" * 8)
        for u, l in tombstones:
            f.write(struct.pack("<QQ", u, l))
        _write_records(f, records)


def read_delta(path: str) -> dict:
    """-> {pshift, chain, index, flags, tombstones: [(u, l)], records: [(ts, fp_hi, fp_lo, bytes)]};
    ValueError for a file that is not a whole delta."""
    with open(path, "rb") as f:
        head = f.read(64)
        if len(head) != 64 or head[:8] != DELTA_MAGIC:
            raise ValueError("not a delta")
        version, pshift, chain, index, flags, nt, nr, total = struct.unpack("<IIQIIQQQ", head[8:56])
        if version != 1:
            raise ValueError("unknown delta version")
        raw = f.read(16 * nt)
        if len(raw) != 16 * nt:
            raise ValueError("truncated tombstones")
        tombs = [struct.unpack("<QQ", raw[16 * i:16 * i + 16]) for i in range(nt)]
        records = _read_records(f, nr)
        if sum(len(r[3]) for r in records) != total or f.read(1) != b"":
            raise ValueError("record bytes do not match the header")
    return dict(pshift=pshift, chain=chain, index=index, flags=flags, tombstones=tombs, records=records)


def valid_deltas(base_path: str):
    """The chain's valid run of deltas after its base, in order: [read_delta(...) of .d1, .d2, ...]."""
    pshift = snapshot.read_snapshot(base_path)[0]
    chain = read_chain_id(base_path)
    out = []
    k = 1
    while chain:
        p = f"{base_path}.d{k}"
        if not os.path.exists(p):
            break
        try:
            d = read_delta(p)
        except ValueError:
            break
        if d["chain"] != chain or d["index"] != k or d["pshift"] != pshift:
            break
        out.append(d)
        k += 1
    return out


def replay_chain(base_path: str):
    """-> ({(u, l): (ts, fp_hi, fp_lo, record_bytes)} of the store the chain's valid run describes,
    deltas applied)."""
    state = {}
    for r in snapshot.read_snapshot(base_path)[2]:
        state[addr_of(r[3])] = r
    deltas = valid_deltas(base_path)
    for d in deltas:
        for a in d["tombstones"]:
            state.pop(a, None)
        for r in d["records"]:
            state[addr_of(r[3])] = r
    return state, len(deltas)
