"""Pages built to reach the branches of the warp LZ4 encoder (lz4_encode_lean).  Test helper, CPU only.

A page is planned sequence by sequence: random literals (datagen's splitmix bytes), then a copy of an
earlier window.  The copy's source is a position the parse has put in its table, so the planner knows
which probe of the search finds it:
  * `resident`: a probe or re-test position of an earlier search (in the table before the batch: the
    batch resolves in the fast path, winner = the planned lane);
  * `batch`: the first probe of the same search (the two lanes share a slot: an alias inside the
    batch, which sends it to lz4_search_slow);
  * `zero`: position 0, which every untouched slot holds on the first search of a page.
The byte before the copy and the byte after it differ from their sources, so the catch-up restores
the planned literal run and the forward extension stops where planned.  Nothing here decides what
the tests count: tests/lz4_trace.py parses every page and the census counts what it saw.

Families (each aims at bins of tests/test_lz4_encoder_census.py):
  lanes      B1, B2, B4  winner lanes, first searches, narrow batches, long searches
  literals   B7, B8      literal runs 0-140 at every anchor & 3, long runs, match codes
  extension  B5, B6      forward extension past every stop lane, backward extension
  ends       B10         the last match against the end margin; every size 13-40
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import datagen
import lz4_trace as T

RING_ACCELS = (1, 4, 12)
RING_MAX_ACCEL = 12
PLAIN_ACCELS = (13, 17)
ACCELS = RING_ACCELS + PLAIN_ACCELS


@dataclass
class Page:
    family: str
    name: str
    accel: int
    page: np.ndarray

    @property
    def n(self) -> int:
        return len(self.page)


class Rng:
    def __init__(self, seed: int):
        self.w = datagen.words(seed, 1 << 14).tolist()
        self.i = 0

    def __call__(self, k: int) -> int:
        self.i += 1
        return self.w[self.i % len(self.w)] % k


class Planner:
    """One page of n bytes, planned for one acceleration."""

    def __init__(self, n: int, accel: int, seed: int):
        self.n, self.accel = n, accel
        self.page = bytearray(datagen.rand_bytes(seed, n).tobytes())
        self.A, self.first, self.prevD = 0, True, 0
        self.resident: list = []
        self.table: dict = {}
        self.rng = Rng(seed ^ 0x5EED)

    @property
    def mflimit(self) -> int:
        return self.n - T.MFLIMIT

    def P(self, k: int) -> int:
        return self.A + 1 + T.probe_off(k, self.accel)

    def k_at(self, pos: int) -> int:
        """The first probe index whose position is >= pos."""
        k = 0
        while self.P(k) < pos:
            k += 1
        return k

    def h(self, q: int) -> int:
        b = bytes(self.page[q:q + 8]).ljust(8, b"\0")
        if self.n >= T.LIMIT64K:
            return ((int.from_bytes(b, "little") << 24) * 889523592379 & (1 << 64) - 1) >> 52
        return (int.from_bytes(b[:4], "little") * 2654435761 & 0xFFFFFFFF) >> 19

    def _residents(self, before: int) -> list:
        """Positions the table holds now (as far as the plan knows), newest first."""
        out = []
        for c in reversed(self.resident[-64:]):
            if c + 8 <= before and self.table.get(self.h(c)) == c and c not in out:
                out.append(c)
        return out

    def seq(self, k: int, back: int, fwd: int, src="resident", end_at: int | None = None) -> bool:
        """Plans one sequence: hit at probe k (-1 = the re-test), `back` bytes of catch-up, `fwd` bytes of
        forward extension past hit + 4 (or the match ending at `end_at`).  src: "resident", "batch",
        "zero", "refill" (the refill position end - 2 of the same batch), "retest" (its re-test
        position) or a position the table holds.  False when it does not fit."""
        A, pg = self.A, self.page
        p = A if k < 0 else self.P(k)
        if k < 0 and self.first:
            return False
        if src == "zero" or (self.first and src == "resident"):
            cands = [0]
        elif src == "batch" and k >= 1:
            cands = [self.P(0)]
        elif src in ("refill", "retest"):
            if self.first:
                return False
            cands = [A - 2 if src == "refill" else A]
        elif isinstance(src, int):
            cands = [src] if self.table.get(self.h(src), 0) == src else []
        else:
            cands = self._residents(A - 2)
            r = self.rng(4)
            cands = cands[r:] + cands[:r]
        stored = [] if self.first else [A - 2, A]
        stored += [self.P(j) for j in range(k + 1)] if k >= 0 else []
        for c in cands[:48]:
            keep = bytes(pg)
            if self._place(k, p, c, back, fwd, end_at) and (src != "resident" or self._found_at(k, p, c, stored)):
                for q in stored:
                    self.table[self.h(q)] = q
                self.resident += stored
                self.A, self.first, self.prevD = self.last_end, False, p - c
                return True
            pg[:] = keep
        return False

    def _found_at(self, k, p, c, stored) -> bool:
        """The copy from table position c is not found before probe k: no earlier store of this batch
        shares its slot, and no earlier probe inside the copy finds an equal word in the table."""
        before = stored[:-1] if k >= 0 else stored[:1]
        if self.h(c) in {self.h(q) for q in before}:
            return False
        for j in range(max(k, 0)):
            q = self.P(j)
            if q >= self.A + 1 and q < p:
                t = self.table.get(self.h(q))
                if t is not None and self.page[t:t + 4] == self.page[q:q + 4]:
                    return False
        return True

    def reject(self, k: int, c: int) -> bool:
        """Gives probe k (-1 = the re-test) the 4 bytes of table position c, more than 65 535 bytes back:
        an equal candidate that the search must pass over.  The anchor stays."""
        p, pg = (self.A if k < 0 else self.P(k)), self.page
        if self.table.get(self.h(c), 0) != c or p + 5 > self.n:
            return False
        if k < 0 and self.prevD and pg[c] == pg[self.A - self.prevD]:
            return False
        w = 5 if self.n >= T.LIMIT64K else 4              # the bytes the slot's hash reads
        if p + w + 1 > self.n:
            return False
        pg[p:p + w] = pg[c:c + w]
        if pg[p + w] == pg[c + w]:
            pg[p + w] ^= 0x5A
        return True

    def _place(self, k, p, c, back, fwd, end_at) -> bool:
        """Writes the copy of the sequence at source c into the page; False when it does not fit."""
        A, pg = self.A, self.page
        back = min(back, p - A)
        S = p - back
        D = p - c
        if D <= 0 or S - D < 0:
            return False
        if end_at is not None:
            fwd = end_at - p - T.MIN_MATCH
        M = back + T.MIN_MATCH + fwd
        if fwd < 0 or S + M > self.n - T.LASTLITERALS or (k >= 0 and self.P(k + 1) > self.mflimit) or A > self.mflimit:
            return False
        # the previous match stops at A because pg[A] differs from its source byte: keep it so
        stop = pg[A - self.prevD] if self.prevD else None
        if S == A and stop is not None and pg[S - D] == stop:
            return False
        if S > A and pg[S - 1] == pg[S - 1 - D]:
            pg[S - 1] = next(v for v in (0x5A, 0xA5, 0x3C) if v != pg[S - 1 - D] and (S - 1 > A or v != stop))
        for i in range(M):
            pg[S + i] = pg[S + i - D]
        if S + M < self.n and pg[S + M] == pg[S + M - D]:
            pg[S + M] ^= 0xA5
        self.last_end = S + M
        return True

    def done(self) -> np.ndarray:
        return np.frombuffer(bytes(self.page), dtype=np.uint8).copy()


LONG_PROBES = list(range(30, 64)) + [64, 65, 127, 128, 129, 192, 200, 260]


def fam_lanes(accel: int, n: int, seed: int, pages: int) -> list:
    """Runs of calm batches (hits at lanes 2-11) that narrow the batch, each followed by a target:
    every lane 1-31, the long probes, or a search that runs into the end margin."""
    out = []
    targets = [-1] + list(range(0, 30)) + LONG_PROBES
    t = seed % len(targets)
    for pi in range(pages):
        pl = Planner(n, accel, seed * 131 + pi)
        pl.seq(pl.rng(10), 0, pl.rng(4), "zero")
        while True:
            calm = 8 + pl.rng(3)
            ok = all(pl.seq(pl.rng(10), 0, pl.rng(4)) for _ in range(calm))
            if not ok or not pl.seq(targets[t % len(targets)], 0, pl.rng(4)):
                break
            t += 1
        while pl.seq(pl.rng(3), 0, 0):       # calm to the end: narrow batches cut by the end margin
            pass
        out.append(Page("lanes", f"lanes.a{accel}.n{n}.{pi}", accel, pl.done()))
    return out


def fam_first(accel: int, seed: int) -> list:
    """The first search of a page hits at every probe lane 2-31 and beyond (the special lanes off)."""
    out = []
    for k in list(range(0, 30)) + [30, 40, 64]:
        for r in range(6):
            pl = Planner(4096, accel, seed + 97 * k + r)
            if pl.seq(k, 0, 8 + r, "zero"):
                pl.seq(-1, 0, 4096, "resident", end_at=pl.n - T.LASTLITERALS)
                out.append(Page("first", f"first.a{accel}.k{k}.{r}", accel, pl.done()))
    return out


def _run_seq(pl: Planner, L: int, fwd: int = 0, src: str = "batch", next_align: int | None = None) -> bool:
    """A sequence with a literal run of exactly L: the first probe at or past anchor + L finds the copy
    and the catch-up walks back to anchor + L.  next_align: fwd is raised by 0-3 so that the next
    sequence's anchor & 3 is next_align."""
    if L == 0:
        k, back = (-1, 0) if not pl.first else (1, 2)
        src = "resident" if k < 0 else "batch"
    else:
        k = pl.k_at(pl.A + L)
        if src == "batch" and k == 0:
            k = 1
        back = pl.P(k) - pl.A - L
    if next_align is not None:
        p = pl.A if k < 0 else pl.P(k)
        fwd += (next_align - (p + T.MIN_MATCH + fwd)) % 4
    return pl.seq(k, back, fwd, src)


def _pack(family: str, accel: int, n: int, seed: int, items, do) -> list:
    """Plans items one after the other into pages of n bytes: do(planner, item) -> bool.  An item that
    does not fit where the page stands gets a filler sequence first, then a fresh page."""
    out, pl = [], None
    for it in items:
        for attempt in range(3):
            if pl is None:
                pl = Planner(n, accel, seed + 7919 * len(out))
                pl.seq(1, 0, 3, "zero")
            if do(pl, it):
                break
            if attempt == 0 and _run_seq(pl, 40 + pl.rng(30), pl.rng(4)):
                continue
            out.append(Page(family, f"{family}.a{accel}.n{n}.{len(out)}", accel, pl.done()))
            pl = None
    if pl is not None:
        out.append(Page(family, f"{family}.a{accel}.n{n}.{len(out)}", accel, pl.done()))
    return out


MCS = [14, 15, 16, 268, 269, 270, 271, 524, 525]


def fam_literals(accel: int, n: int, seed: int) -> list:
    """Literal runs 0-140 at every anchor & 3 (twice), runs of 255-258, 269-271, 1000+, and the match
    codes 14-16, 268-271, 524, 525 after runs <= 128 and of 129."""
    items = [("run", L, a) for L in range(141) for a in range(4)] * 3
    items += [("run", L, L % 4) for L in (255, 256, 257, 258, 269, 270, 271, 1000, 1500)] * 2
    items += [("mc", 5 + 37 * i % 120, mc) for i, mc in enumerate(MCS * 3)] + [("mc", 129, mc) for mc in MCS * 3]

    def do(pl, it):
        kind, a, b = it
        if kind == "run":      # a short sequence whose end puts the run's anchor at & 3 == b
            return _run_seq(pl, 3, 0, next_align=b) and _run_seq(pl, a, pl.rng(4))
        return _mc_seq(pl, a, b)
    return _pack("literals", accel, n, seed, items, do)


def _mc_seq(pl: Planner, L: int, mc: int) -> bool:
    k = pl.k_at(pl.A + L)
    k = max(k, 1)
    back = pl.P(k) - pl.A - L
    return back <= mc and pl.seq(k, back, mc - back, "batch")


def fam_extension(accel: int, n: int, seed: int) -> list:
    """Forward extensions of 3-35 bytes, past every 16-byte lane of the first 512-byte step and of a
    later one; backward extensions of 0-40 bytes and ~100, stopped by the anchor or by the literal
    before the copy."""
    items = [("f", F) for F in range(3, 36)] * 2
    items += [("f", 36 + 16 * f + (f * 5) % 16) for f in range(32)] * 2
    items += [("f", 548 + 16 * f + (f * 7) % 16) for f in range(32)] * 2
    items += [("b", b) for b in list(range(0, 41)) + [100, 101]] * 3

    def do(pl, it):
        kind, v = it
        if kind == "f":
            return pl.seq(pl.rng(10), 0, v)
        k = pl.k_at(pl.A + v + 1 + pl.rng(8))    # the copy starts inside the literals: back = v
        return pl.seq(k, v, pl.rng(4), "zero" if pl.first else "batch" if k > 0 else "resident")
    return _pack("extension", accel, n, seed, items, do)


def fam_ends(accel: int, n: int, seed: int) -> list:
    """A last match that ends at mflimit - 1, mflimit, mflimit + 1 and mlimit, after a few sequences
    (small pages: straight away); the page before it is random literals."""
    out = []
    mflimit, mlimit = n - T.MFLIMIT, n - T.LASTLITERALS
    for e in (mflimit - 1, mflimit, mflimit + 1, mlimit):
        for r in range(3):
            pl = Planner(n, accel, seed + 31 * e + r)
            if n >= 4096:
                while pl.A < n - 3000 and _run_seq(pl, 20 + pl.rng(60), pl.rng(40)):
                    pass
            for k in range(0, 40):           # the first probe from which a match ending at e fits
                if pl.seq(k, 0, 0, "zero" if pl.first else "resident", end_at=e):
                    break
            out.append(Page("ends", f"ends.a{accel}.n{n}.e{e - n}.{r}", accel, pl.done()))
    return out


def _land(pl: Planner, end: int) -> bool:
    """One sequence (a short literal run, then a copy with a short period) that ends at `end`."""
    for k in range(1, 6):
        if pl.seq(k, 0, 0, "zero" if pl.first else "batch", end_at=end):
            return True
    return False


def fam_aliases(accel: int, n: int, seed: int) -> list:
    """Certain aliases with the special lanes: the re-test finds the refill (lane 0 + lane 1, a
    period of 2 across the end of the match), and a probe finds the refill or the re-test position
    of its own batch (lane 0 or 1 + a probe lane)."""
    items = [("refill", -1), ("refill", 2), ("refill", 9), ("retest", 3), ("retest", 11)] * 12

    def do(pl, it):
        src, k = it
        return _run_seq(pl, 20 + pl.rng(20), pl.rng(4)) and pl.seq(k, 0, 1 + pl.rng(6), src)
    return _pack("aliases", accel, n, seed, items, do)


def fam_guards(accel: int, seed: int) -> list:
    """The bounds of the fast path's long catch-up, `ip >= anchor + 5 && match >= 5`, at back = 4:
    a hit 4 bytes past the anchor (accel 1 and 2: probe positions anchor + 1, 2, 3, 4), and a hit
    whose candidate is position 4 (refilled behind a first match that ends at 6, one batch earlier)."""
    out = []
    for r in range(12):
        pl = Planner(65536, accel, seed + r)
        pl.seq(200, 0, 3, "zero")                     # a long first search: its late probes are 3-4 apart
        sparse = [c for c in pl.resident if not {c - 1, c - 2, c - 3} & set(pl.resident)]
        got = tries = 0
        while got < 4 and tries < 60 and _run_seq(pl, 10 + pl.rng(30), pl.rng(4)):
            tries += 1
            k = next(j for j in range(8) if pl.P(j) >= pl.A + 4)
            # a table position whose three predecessors were never stored: the earlier probes inside the
            # copy find nothing, and the hit at anchor + 4 extends back to the anchor
            if pl.P(k) == pl.A + 4 and pl.seq(k, 4, pl.rng(6), sparse[-1 - (got + tries) % min(20, len(sparse))]):
                got += 1
        _land(pl, pl.n - T.LASTLITERALS)
        out.append(Page("guards", f"guards.a{accel}.anchor4.{r}", accel, pl.done()))
        pl = Planner(4096, 12, seed + 100 + r)
        pl.seq(1, 0, 0, "zero")                        # the match ends at 6: position 4 is refilled
        _run_seq(pl, 10 + r, 0)
        for k in range(2, 6):
            if pl.seq(k, 4, pl.rng(6), 4):
                break
        _land(pl, pl.n - T.LASTLITERALS)
        out.append(Page("guards", f"guards.a12.cand4.{r}", 12, pl.done()))
    return out


def fam_ring(accel: int, n: int, seed: int) -> list:
    """The ring: sequences that jump 256-1279 and more bytes and end at mod 256 in 0-7 or 252-255,
    anchors at 256 g + 3, 4, 5, and literal runs of 120-128 whose speculative words cross the wrap
    of the 1 KiB ring."""
    ends = list(range(8)) + list(range(252, 256))
    items = [("jump", J, t) for J in (256, 512, 768, 1024, 1280) for t in ends] * 3
    items += [("anchor", 0, t) for t in (3, 4, 5)] * 4
    items += [("wrap", L, 0) for L in range(120, 129)] * 3

    def do(pl, it):
        kind, a, b = it
        A = pl.A
        if kind == "jump":
            return _land(pl, A + a + (b - (A + a)) % 256)
        if kind == "anchor":
            return _land(pl, A + 40 + (b - (A + 40)) % 256) and _run_seq(pl, 3 + pl.rng(8), pl.rng(4))
        t = 1024 - a + 1 + pl.rng(a - 1)                  # anchor mod 1024 in (1024 - run, 1024)
        return _land(pl, A + 40 + (t - (A + 40)) % 1024) and _run_seq(pl, a, pl.rng(4))
    return _pack("ring", accel, n, seed, items, do)


def far_finder(k: int) -> str:
    """Who meets a candidate at probe k: the re-test, a lane of the batch (probes 0-29) or
    lz4_search_slow (probes from 30)."""
    return "retest" if k < 0 else "lane" if k < 30 else "slow"


def fam_far(n: int, seed: int) -> list:
    """byU32 pages: a candidate at distance 65 535 (taken) and 65 536, 65 537 (passed over), met by
    the re-test, by a probe lane of the batch and by lz4_search_slow.  The plan does not always
    survive the long landing match, so seeded variants are kept only where the trace confirms the
    event (three per cell)."""
    out = []
    fits = n >= 65536 + 2 * T.MFLIMIT                      # at 65 547 only the re-test at mflimit fits
    for d in (65535, 65536, 65537) if fits else (65535,):
        for finder, k0 in (("retest", -1), ("lane", 5), ("slow", 35)) if fits else (("retest", -1),):
            kept = 0
            for r in range(16):
                if kept == 3:
                    break
                k = k0 if k0 < 0 else k0 + r % 4
                pl = Planner(n, 12, seed + 1000 * d + 10 * k0 + r)
                # (at 65 547 the candidate is position 0 itself: no copy of its bytes may replace it)
                pl.seq(3, 0, 3, "zero") if fits else pl.seq(2, 0, 3, "batch")
                for _ in range(4):
                    pl.seq(pl.rng(6), 0, pl.rng(4))
                cs = pl._residents(pl.A - 2) if fits else [0]
                if not cs:
                    continue
                c = cs[r % len(cs)]
                at = c + d if k < 0 else c + d - 1 - T.probe_off(k, 12)
                if not _land(pl, at):
                    continue
                if d == 65535:
                    ok = pl.seq(k, 0, 1 + pl.rng(3), c)        # 5 equal bytes: hash5 reads 5
                else:
                    ok = pl.reject(k, c) and pl.seq(k + 3 if k >= 0 else 2, 0, pl.rng(4), "batch")
                if not ok:
                    continue
                _land(pl, pl.n - T.LASTLITERALS)
                page = pl.done()
                tr = T.parse(page, 12, lanes=False)
                seen = [(s.probe, s.off) for s in tr.seqs if s.off == d] + [e for s in tr.seqs for e in s.far if e[1] == d]
                if any(far_finder(q) == finder for q, _ in seen):
                    out.append(Page("far", f"far.n{n}.d{d}.{finder}.{r}", 12, page))
                    kept += 1
    return out


def fam_ckpt(n: int, seed: int, pages: int) -> list:
    """Sequences that start at k n/16 and at k n/16 - 1, and matches that cover several sixteenths."""
    out = []
    S = n // 16
    for r in range(pages):
        pl = Planner(n, 12, seed + r)
        k = 1
        while k < 16:
            skip = 3 if k % 5 == 4 else 1                  # now and then a match over several sixteenths
            e = (k + skip - 1) * S - (k + r) % 2
            if e > pl.A and _land(pl, e):
                _run_seq(pl, 1 + pl.rng(3), pl.rng(3)) if S >= 64 else None
            k += skip
        _land(pl, pl.n - T.LASTLITERALS)
        out.append(Page("ckpt", f"ckpt.n{n}.{r}", 12, pl.done()))
    return out


CODEC_SIZES = list(range(13, 41)) + [300, 4096, 4099, 16384, 65536, 65546, 65547, 131072]
STORE_SIZES = [1 << s for s in (6, 8, 10, 12, 16, 17, 18)]


def corpus() -> list:
    """The whole corpus, deterministic: a list of Page."""
    out = []
    for a in ACCELS:
        out += fam_first(a, 100 + a)
        out += fam_lanes(a, 65536, 200 + a, 3 if a < 12 else 9)
        out += fam_lanes(a, 16384, 300 + a, 2)
    out += fam_lanes(12, 131072, 400, 1) + fam_lanes(1, 131072, 401, 1) + fam_lanes(17, 65547, 402, 1)
    twelve = [p for p in out if p.family == "lanes" and p.accel == 12]
    out += [Page(p.family, p.name.replace(".a12.", ".a12as13."), 13, p.page) for p in twelve]
    out += fam_literals(1, 65536, 500) + fam_literals(13, 65536, 501) + fam_literals(12, 65546, 502)
    out += fam_literals(4, 131072, 503)
    out += fam_extension(12, 65536, 600) + fam_extension(17, 131072, 601) + fam_extension(1, 4099, 602)
    for i, n in enumerate(CODEC_SIZES):
        for a in (1, 12, 13):
            out += fam_ends(a, n, 700 + 10 * i + a)
    for i, n in enumerate((64, 256, 1024)):
        out += fam_ends(12, n, 800 + i) + fam_extension(12, n, 810 + i)
    out += fam_lanes(12, 1 << 18, 820, 1) + fam_extension(12, 1 << 18, 821)
    out += fam_aliases(12, 65536, 900) + fam_aliases(12, 131072, 901) + fam_aliases(1, 16384, 902)
    out += fam_guards(1, 910) + fam_guards(2, 911)
    out += fam_ring(12, 65536, 920) + fam_ring(1, 65536, 921) + fam_ring(4, 16384, 922)
    for i, n in enumerate((65547, 1 << 17, 1 << 18)):
        out += fam_far(n, 930 + i)
    for i, n in enumerate(STORE_SIZES[:-1]):
        out += fam_ckpt(n, 940 + i, 6 if n < 4096 else 3)
    return out
