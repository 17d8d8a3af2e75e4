"""LZ4 blocks written from sequence lists, to reach decoder branches that the encoder's own blocks
may never reach.  Test helper, CPU only.

A block is a list of sequences (literals, offset, match length) and a final literal run; the page it
stands for is what an LZ4_decompress_fast-style decoder makes of it (overlapping copies byte by
byte).  Literal bytes are random, so every match copies bytes that differ from their surroundings.

`cases(n)` returns the families below for a page of n bytes; a family leaves out what does not fit.

  F1 offsets       every offset 1-140, 255, 256, 4095, 4096, 65535 x lengths 4, 15-19, 31-33, 63-65,
                   127-129, 270, 271, 4095-4097, 8175, 8200; the destination's `& 15` rotates
  F2 lengths       literal and match-length fields of 14, 15, 269, 270 (255, 0), 525, 8175 (32 x 255),
                   8430 (33 x 255) and 12000
  F3 chains        matches that copy the previous match's output, 2-40 deep, shifted over the edges of
                   a batch of 32 sequences and over sixteenths of the page
  F4 literals      runs of 0-70 bytes at every destination alignment, and runs of 100, 1000, 5000
  F5 block end     last match ends at n - 5; literals end at n - 9 before a 4-byte match; final run of
                   exactly 5 after a long overlapping match; offset == op
  F6 checkpoints   sequences starting exactly at k n/16 and at k n/16 + n/16 - 1; empty sixteenths
  F7 pair fields   match length - 4 >= 65 536 at offsets 1, 3, 17, 31, 32, 135, 136, 4096; literal
                   runs >= 65 536; matches written above 65 536
  F8 twins         invalid: match ends at n - 4; literals end at n - 8 .. n - 1 before a match;
                   offset == op + 1; offset 0; one trailing byte; truncated length extensions
"""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

import datagen

OFFSETS = list(range(1, 141)) + [255, 256, 4095, 4096, 65535]
LENGTHS = [4, 15, 16, 17, 18, 19, 31, 32, 33, 63, 64, 65, 127, 128, 129, 270, 271, 4095, 4096, 4097, 8175, 8200]
FIELDS = [14, 15, 269, 270, 525, 8175, 8430, 12000]
PAIR_OFFSETS = [1, 3, 17, 31, 32, 135, 136, 4096]


@dataclass
class Case:
    family: str
    name: str
    n: int
    block: bytes
    page: bytes | None          # None: an invalid twin (F8)

    @property
    def valid(self) -> bool:
        return self.page is not None


def _ext(v: int) -> bytes:
    """Length extension of a 4-bit field whose value v is >= 15."""
    v -= 15
    return b"\xff" * (v // 255) + bytes([v % 255])


def encode(seqs, last: bytes) -> bytes:
    """[(literal bytes, offset, match length)] + final literals -> block bytes (no checks)."""
    out = bytearray()
    for lit, off, mlen in seqs:
        ml = mlen - 4
        out.append(min(len(lit), 15) << 4 | min(ml, 15))
        if len(lit) >= 15:
            out += _ext(len(lit))
        out += lit
        out += struct.pack("<H", off)
        if ml >= 15:
            out += _ext(ml)
    out.append(min(len(last), 15) << 4)
    if len(last) >= 15:
        out += _ext(len(last))
    out += last
    return bytes(out)


class Builder:
    """One block of a page of n bytes, built sequence by sequence."""

    def __init__(self, n: int, seed: int):
        self.n, self.op = n, 0
        self.pool = datagen.rand_bytes(seed, n)         # literal at page position p is pool[p]
        self.page = np.zeros(n, dtype=np.uint8)
        self.seqs = []

    def fits(self, lit: int, mlen: int) -> bool:
        return self.op + lit + mlen + 5 <= self.n       # the match ends at n - 5 at the latest

    def lits(self, k: int) -> bytes:
        b = self.pool[self.op:self.op + k]
        self.page[self.op:self.op + k] = b
        self.op += k
        return b.tobytes()

    def copy(self, off: int, mlen: int) -> None:
        op = self.op
        if off >= mlen:
            self.page[op:op + mlen] = self.page[op - off:op - off + mlen]
        else:                                           # overlapping: the last `off` bytes repeat
            self.page[op:op + mlen] = np.resize(self.page[op - off:op], mlen)
        self.op += mlen

    def seq(self, lit: int, off: int, mlen: int) -> None:
        assert self.fits(lit, mlen) and 1 <= off <= self.op + lit and mlen >= 4, (self.n, self.op, lit, off, mlen)
        b = self.lits(lit)
        self.copy(off, mlen)
        self.seqs.append((b, off, mlen))

    def lit_for(self, off: int, align: int) -> int:
        """The fewest literals that put the match source in the page and its destination at `& 15 == align`."""
        k = max(0, off - self.op)
        return k + (align - (self.op + k)) % 16

    def finish(self) -> tuple[bytes, bytes]:
        rest = self.n - self.op
        if rest > 64 and self.op:
            # one long match before 16 final literals: a long final run's extension bytes would make
            # the block longer than the n + 1024 bytes a store keeps (filemap.c:120)
            self.seq(1, min(self.op + 1, 1000), rest - 17)
        last = self.lits(self.n - self.op)
        return encode(self.seqs, last), self.page.tobytes()


def _pack(n: int, seed: int, family: str, items) -> list[Case]:
    """Items (offset, match length, destination alignment) greedily into as many blocks as they need;
    an item that does not fit an empty block is left out."""
    out, b = [], None
    for off, mlen, align in items:
        if b is None or not b.fits(b.lit_for(off, align), mlen):
            fresh = Builder(n, seed + 7919 * len(out))
            if not fresh.fits(fresh.lit_for(off, align), mlen):
                continue
            if b is not None and b.seqs:
                out.append(Case(family, f"{family}.{len(out)}", n, *b.finish()))
            b = fresh
        b.seq(b.lit_for(off, align), off, mlen)
    if b is not None and b.seqs:
        out.append(Case(family, f"{family}.{len(out)}", n, *b.finish()))
    return out


def f1_offsets(n: int) -> list[Case]:
    items = [(off, mlen, (i * 5 + j) % 16) for i, off in enumerate(OFFSETS) for j, mlen in enumerate(LENGTHS)]
    return _pack(n, 1000 + n, "F1", items)


def f2_lengths(n: int) -> list[Case]:
    out = []
    for i, v in enumerate(FIELDS):
        b = Builder(n, 2000 + n + i)
        if b.fits(v, 4):                                # literal field v
            b.seq(v, 1 + i, 4)
        b2 = Builder(n, 2100 + n + i)
        if b2.fits(3, v + 4):                           # match field v (match length v + 4)
            b2.seq(3, 3 if i % 2 else 1, v + 4)
        for name, x in ((f"F2.lit{v}", b), (f"F2.match{v}", b2)):
            if x.seqs:
                out.append(Case("F2", name, n, *x.finish()))
    return out


def f3_chains(n: int) -> list[Case]:
    out = []
    for depth in (2, 8, 31, 32, 40):
        for skew in (0, 1, 15, 31, 33):
            b = Builder(n, 3000 + n + 64 * depth + skew)
            if not b.fits(16, 4):
                continue
            b.seq(16, 16, 4)
            for _ in range(skew):                       # independent sequences before the chain
                if not b.fits(1, 4):
                    break
                b.seq(1, 13, 4)
            prev = 4
            for j in range(depth):                      # each match starts its source in the previous match
                lit, mlen = j % 3, 4 + (j * 7) % 13
                if not b.fits(lit, mlen):
                    break
                b.seq(lit, lit + prev - j % 2, mlen)
                prev = mlen
            out.append(Case("F3", f"F3.d{depth}s{skew}", n, *b.finish()))
    # a chain across each sixteenth's edge
    S = n // 16
    b = Builder(n, 3900 + n)
    for k in range(1, 16):
        start = k * S - 6
        if start <= b.op or not b.fits(start - b.op, 4):
            continue
        b.seq(start - b.op, min(start, 1 + k % 7), 4)
        prev = 4
        for j in range(6):
            if not b.fits(1, 5):
                break
            b.seq(1, 1 + prev, 5)
            prev = 5
    if b.seqs:
        out.append(Case("F3", "F3.edges", n, *b.finish()))
    return out


def f4_literals(n: int) -> list[Case]:
    out, b = [], None
    runs = [(L, a) for L in range(71) for a in range(16)] + [(L, a) for L in (100, 1000, 5000) for a in (0, 7)]
    for L, a in runs:
        for _ in range(2):
            if b is None:
                b = Builder(n, 4000 + n + len(out))
                if b.fits(8, 4):
                    b.seq(8, 8, 4)
            pad = 4 + (a - b.op - 4) % 16                # a match of 4-19 bytes puts the run at `& 15 == a`
            if b.seqs and b.fits(L, pad + 4):
                b.seq(0, 1, pad)
                b.seq(L, 4, 4)
                break
            if len(b.seqs) > 1:
                out.append(Case("F4", f"F4.{len(out)}", n, *b.finish()))
            b = None
    if b is not None and len(b.seqs) > 1:
        out.append(Case("F4", f"F4.{len(out)}", n, *b.finish()))
    return out


def f5_block_end(n: int) -> list[Case]:
    out = []
    b = Builder(n, 5000 + n)
    if b.fits(7, n - 12):
        b.seq(7, 3, n - 12)                             # match ends at n - 5
        out.append(Case("F5", "F5.match_to_n-5", n, *b.finish()))
    b = Builder(n, 5001 + n)
    if n >= 13:
        if n > 64:                                      # (a long match first keeps the block short)
            b.seq(9, 9, n - 50)
        b.seq(n - 9 - b.op, 9, 4)                       # literals end at n - 9, 4-byte match
        out.append(Case("F5", "F5.lits_to_n-9", n, *b.finish()))
    b = Builder(n, 5002 + n)
    if n >= 24:
        b.seq(2, 2, n - 2 - 5 - 9)
        b.seq(0, 5, 9)                                  # final run of exactly 5
        out.append(Case("F5", "F5.last_run_5", n, *b.finish()))
    for L in (1, 4, 16, 33, 200):
        b = Builder(n, 5010 + n + L)
        if b.fits(L, 4):
            b.seq(L, L, min(4 + L, n - L - 5))          # offset == op: copies from page position 0
            out.append(Case("F5", f"F5.off_eq_op{L}", n, *b.finish()))
    return out


def f6_checkpoints(n: int) -> list[Case]:
    """Sequences (lit 0) whose literal start lands at distance d into sixteenth k: d = 0 and d = S - 1
    (the largest distance a word holds), and every third sixteenth only (the others stay empty)."""
    S, out = n // 16, []
    for variant, ks, d in (("start", range(1, 16), 0), ("end", range(1, 16), S - 1), ("sparse", range(1, 16, 3), S - 1)):
        b = Builder(n, 6000 + n + len(variant))
        if not b.fits(1, 4):
            continue
        b.seq(1, 1, 4)
        for k in ks:
            gap = k * S + d - b.op
            if gap >= 4 and b.fits(0, gap):
                b.seq(0, min(b.op, 1 + k % 5), gap)
        out.append(Case("F6", f"F6.{variant}", n, *b.finish()))
    return out


def f7_pair(n: int) -> list[Case]:
    out = _pack(n, 7000 + n, "F7", [(off, 65540 + 2 * i, i % 16) for i, off in enumerate(PAIR_OFFSETS)])
    b = Builder(n, 7100 + n)
    if b.fits(65536 + 3, 4):
        b.seq(65536 + 3, 17, 4)                         # literal run >= 65 536
        for off, mlen in ((1, 40), (31, 100), (136, 300), (4096, 5000), (65535, 70)):
            if b.fits(1, mlen):
                b.seq(1, off, mlen)                     # destinations above 65 536
        out.append(Case("F7", "F7.long_lits", n, *b.finish()))
    return out


def f8_twins(n: int) -> list[Case]:
    out = []

    def twin(name, seqs, last):
        out.append(Case("F8", f"F8.{name}", n, encode(seqs, last), None))

    r = datagen.rand_bytes(8000 + n, n + 64).tobytes()
    if n >= 16:
        twin("match_to_n-4", [(r[:4], 2, n - 8)], r[4:8])
    for j in range(8):                                  # literals end at n - 8 + j, then a match
        k = n - 8 + j
        if k > 64:
            twin(f"lits_to_n-{8 - j}", [(r[:8], 8, k - 40), (r[8:40], 1, 4)], r[k:max(k, n - 4)])
        elif k >= 1:
            twin(f"lits_to_n-{8 - j}", [(r[:k], 1, 4)], r[k:max(k, n - 4)])
    if n >= 16:
        # after the first sequence: one long match and 16 literals, or the rest as literals
        rest = ([(r[:1], 1, n - 26)], r[:16]) if n > 64 else ([], r[5:n - 4])
        twin("off_eq_op+1", [(r[:5], 6, 4)] + rest[0], rest[1])
        twin("off_0", [(r[:5], 0, 4)] + rest[0], rest[1])
        out.append(Case("F8", "F8.trailing_byte", n, encode([(r[:5], 5, 4)] + rest[0], rest[1]) + b"\x00", None))
    out.append(Case("F8", "F8.trunc_lit_ext", n, b"\xf0" + b"\xff" * 40, None))
    out.append(Case("F8", "F8.trunc_lit_ext0", n, b"\xf0", None))
    if n >= 32:
        out.append(Case("F8", "F8.trunc_match_ext", n, b"\x1f" + r[:1] + b"\x01\x00" + b"\xff" * 3, None))
    return out


FAMILIES = (f1_offsets, f2_lengths, f3_chains, f4_literals, f5_block_end, f6_checkpoints, f7_pair, f8_twins)


def cases(n: int, families=FAMILIES) -> list[Case]:
    return [c for f in families for c in f(n)]
