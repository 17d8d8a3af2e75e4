"""The reference LZ4 parse, traced sequence by sequence, and the warp encoder's view of each sequence.
Test helper, CPU only.

`parse(page, accel)` is an independent Python statement of LZ4 1.8.1's LZ4_compress_generic as
oracle/lz4_block.c states it: byU16 with the 13-bit hash4 below 65 547 bytes, byU32 with the 12-bit
hash5 and the MAX_DISTANCE test from 65 547 bytes; the acceleration step schedule (a step of 1, then
64 probes at `accel`, 64 at `accel + 1`, ...); MFLIMIT 12 and LASTLITERALS 5; after a match, the table
refill of `end - 2` and the immediate re-test at `end`.  It is exact: `Trace.block()` rebuilds the
block from the sequences (lz4_synth.encode writes it) and must equal oracle.lz4_encode.

Each sequence also carries its batch as lz4_encode_lean (edge_fuse_b200/csrc/lz4_encode_ring.cuh)
lays it out.  This lane model is read off the kernel's code, not derived from the parse:
  * lanes (lz4_encode_ring.cuh:244-255): lane 0 at end - 2 (the refill), lane 1 at end (the
    re-test), lane j >= 2 at end + 1 + lz4_probe_off(j - 2, accel); the first search of a page is the
    same batch with end = 0 and lanes 0 and 1 switched off;
  * a probe lane takes part while end + 2 + accel (j - 2) <= mflimit (`en_below`, :247-251), and
    only below the batch width (:321);
  * every enabled lane reads its slot, stores its position, reads the slot back (:326-334); a lane
    hits when the slot's old position holds its 4 bytes (byU32: within 65 535 bytes) (:364-366); a
    lane whose read-back is not its own position is foreign (:364);
  * the batch resolves in the fast path when the lowest hit lies below the lowest foreign lane
    (:382), else through lz4_search_slow (:406-429): from slot 0 when a lane is foreign, from the
    batch width when every lane was held back by nothing but the width, else the search ran into
    the end margin;
  * the width state (:263-265, :393-394, :411-412): a fast path with winner w < 12 counts one more
    calm batch, eight in a row make the next batches 16 lanes wide; a winner at lane >= 12 or any
    slow path resets to 32 lanes.

Which lane's store wins when two enabled lanes share a slot is not defined by the hardware.  Where
that decides the path (an alias that straddles the winner) the batch is `ambiguous`, and the width
state is unknown until the next batch that resets it whatever it was.  `simulate` never guesses.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

MIN_MATCH, LASTLITERALS, MFLIMIT, MIN_INPUT = 4, 5, 12, 13
LIMIT64K, FAR, SKIP = 65536 + 11, 65535, 6
LANES, NARROW_W, NARROW_HIT, CALM = 32, 16, 12, 8


def probe_off(k: int, accel: int) -> int:
    """Offset of probe k of a search from its first probe position (lz4_probe_off)."""
    if k == 0:
        return 0
    m = k - 1
    q, r = m >> 6, m & 63
    return 1 + accel * m + 32 * q * (q - 1) + q * r


def _hashes(page: bytes, wide: bool):
    a = np.frombuffer(page + b"\0" * 8, dtype=np.uint8).astype(np.uint64)
    n = len(page)
    w64 = np.zeros(n + 1, dtype=np.uint64)
    for i in range(8):
        w64 |= a[i:i + n + 1] << np.uint64(8 * i)
    w32 = w64 & np.uint64(0xFFFFFFFF)
    with np.errstate(over="ignore"):
        if wide:
            h = ((w64 << np.uint64(24)) * np.uint64(889523592379)) >> np.uint64(52)
        else:
            h = ((w32 * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(19)
    return h.astype(np.int64).tolist(), w32.astype(np.int64).tolist()


def _common(b: bytes, a: int, m: int, lim: int) -> int:
    n = 0
    while a + n + 64 <= lim and b[a + n:a + n + 64] == b[m + n:m + n + 64]:
        n += 64
    while a + n < lim and b[a + n] == b[m + n]:
        n += 1
    return n


@dataclass
class Seq:
    anchor: int          # first literal of the sequence
    start: int           # end of the previous match (the re-test position); 0 on the first search
    first: bool          # the first search of the page (lanes 0 and 1 off)
    probe: int           # probe index of the hit, -1 = the re-test
    hit: int             # position of the hit before the catch-up
    cand: int            # its candidate
    back: int            # backward extension (catch-up)
    fwd: int             # common length past hit + 4
    lit: int             # literal run
    off: int
    # the batch (lanes 0..31)
    lane: int            # lane of the hit, -1 when it lies beyond lane 31
    en: int = 0          # lanes enabled by the end margin (and, for 0/1, by the page having started)
    hits: int = 0        # lanes whose old slot value holds their 4 bytes
    slots: list = field(default_factory=list)
    far: list = field(default_factory=list)   # (probe, distance): equal candidates passed over as too far

    @property
    def mc(self) -> int:
        return self.back + self.fwd

    @property
    def ip(self) -> int:
        return self.hit - self.back

    @property
    def end(self) -> int:
        return self.hit + MIN_MATCH + self.fwd


@dataclass
class Trace:
    n: int
    accel: int
    wide: bool
    seqs: list
    last: int                    # anchor of the last literals
    tail_batch: Seq | None       # the batch of a search that ran into the end margin (lane = -1)
    tail_probes: int             # probes that search made before the margin
    page: bytes = b""

    @property
    def mflimit(self) -> int:
        return self.n - MFLIMIT

    @property
    def mlimit(self) -> int:
        return self.n - LASTLITERALS

    def block(self) -> bytes:
        import lz4_synth
        p = self.page
        return lz4_synth.encode([(p[s.anchor:s.ip], s.off, s.mc + MIN_MATCH) for s in self.seqs], p[self.last:])


def _batch(s: Seq, anchor: int, first: bool, accel: int, mflimit: int, hsh, w32, table, pre, wide: bool) -> None:
    """Fills the batch fields of s: lane positions, margin enables, slots, hits on the old slot values."""
    en = hits = 0
    slots = [-1] * LANES
    for j in range(LANES):
        if j < 2:
            if first:
                continue
            pos = anchor - 2 + 2 * j
        else:
            if anchor + 2 + accel * (j - 2) > mflimit:
                continue
            pos = anchor + 1 + probe_off(j - 2, accel)
        en |= 1 << j
        h = hsh[pos]
        slots[j] = h
        c = pre.get(h, table[h])
        if j and w32[c] == w32[pos] and (not wide or c + FAR >= pos):
            hits |= 1 << j
    s.en, s.hits, s.slots = en, hits, slots


def parse(page, accel: int = 12, lanes: bool = True) -> Trace:
    page = bytes(np.ascontiguousarray(page, dtype=np.uint8))
    n = len(page)
    accel = max(1, accel)
    wide = n >= LIMIT64K
    tr = Trace(n, accel, wide, [], 0, None, 0, page)
    if n < MIN_INPUT:
        return tr
    mflimit, mlimit = n - MFLIMIT, n - LASTLITERALS
    hsh, w32 = _hashes(page, wide)
    table = [0] * 8192
    pre: dict = {}

    def put(h, v):
        if h not in pre:
            pre[h] = table[h]
        table[h] = v

    anchor = 0
    first = True
    while True:
        pre.clear()
        far = []
        probe, ip, match = -2, 0, 0
        if not first:                                   # refill and re-test (lz4.c:691-707)
            put(hsh[anchor - 2], anchor - 2)
            h = hsh[anchor]
            match = table[h]
            put(h, anchor)
            if w32[match] == w32[anchor]:
                if match + FAR >= anchor:
                    probe, ip = -1, anchor
                else:
                    far.append((-1, anchor - match))
        if probe == -2:                                 # the search (lz4.c:593-619)
            p0 = 1 if first else anchor + 1
            fwd, step, nb, k = p0, 1, accel << SKIP, 0
            while True:
                ip = fwd
                fwd += step
                step = nb >> SKIP
                nb += 1
                if fwd > mflimit:
                    break
                h = hsh[ip]
                match = table[h]
                put(h, ip)
                if w32[match] == w32[ip]:
                    if not (wide and match + FAR < ip):
                        probe = k
                        break
                    far.append((k, ip - match))
                k += 1
            if probe == -2:                             # ran into the end margin
                if lanes:
                    t = Seq(anchor, 0 if first else anchor, first, -2, 0, 0, 0, 0, 0, 0, -1)
                    _batch(t, anchor, first, accel, mflimit, hsh, w32, table, pre, wide)
                    t.far = far
                    tr.tail_batch, tr.tail_probes = t, k
                break
        back = 0
        if probe >= 0:                                  # catch-up (lz4.c:622)
            while ip - back > anchor and match - back > 0 and page[ip - back - 1] == page[match - back - 1]:
                back += 1
        f = _common(page, ip + MIN_MATCH, match + MIN_MATCH, mlimit)
        lane = 1 if probe == -1 else (probe + 2 if probe < LANES - 2 else -1)
        s = Seq(anchor, 0 if first else anchor, first, probe, ip, match, back, f, ip - back - anchor, ip - match, lane)
        s.far = far
        if lanes:
            _batch(s, anchor, first, accel, mflimit, hsh, w32, table, pre, wide)
        tr.seqs.append(s)
        anchor = s.end
        first = False
        if anchor > mflimit:
            break
    tr.last = anchor
    return tr


# ---- the width / calm state machine -------------------------------------------------------------

@dataclass
class Step:
    width: int | None        # batch width the sequence was searched with, None = unknown
    path: str                # "fast", "slow0" (foreign lane), "slow_w" (probes exhausted), "end", "ambiguous", "unknown"
    narrow_cut: bool = False  # a narrow batch with lanes cut by the end margin


def _alias_groups(en: int, slots) -> list:
    groups: dict = {}
    for j in range(LANES):
        if en >> j & 1:
            groups.setdefault(slots[j], []).append(j)
    return [g for g in groups.values() if len(g) > 1]


def resolve(s: Seq, width: int) -> tuple[str, int]:
    """Path of one batch at a known width -> (path, w) with w the fast-path winner.  path is "fast",
    "slow0", "slow_w", "end" or "ambiguous"."""
    wmask = (1 << width) - 1
    en = s.en & wmask
    hits = s.hits & en
    low = (hits & -hits).bit_length() - 1 if hits else LANES
    groups = _alias_groups(en, s.slots)
    if not hits:
        if groups:
            return "slow0", -1
        full = all((s.en >> j & 1) or j >= width or j < 2 for j in range(LANES))
        return ("slow_w" if full else "end"), -1
    certain_slow = any(g[1] <= low for g in groups)       # two lanes of one slot at or below the winner
    if certain_slow:
        return "slow0", -1
    if any(g[0] <= low for g in groups):                  # straddles the winner: whose store wins decides
        return "ambiguous", low
    return "fast", low


def simulate(tr: Trace) -> list:
    """One Step per sequence (and one for the tail batch, if any, last)."""
    out = []
    width, calm = LANES, 0
    known = True
    batches = tr.seqs + ([tr.tail_batch] if tr.tail_batch is not None else [])
    for s in batches:
        if not known:
            # a batch resets the state whatever the width was when its winner is at lane >= 12, it has
            # none, or two lanes alias at or below the winner at both widths
            r16, r32 = resolve(s, NARROW_W), resolve(s, LANES)
            resets = all(p in ("slow0", "slow_w", "end") or (p == "fast" and w >= NARROW_HIT) for p, w in (r16, r32))
            same = r16[0] == r32[0] and r16[0] != "ambiguous"
            out.append(Step(None, r16[0] if same else "unknown"))   # the path, where both widths agree
            if resets:
                known, width, calm = True, LANES, 0
            continue
        path, w = resolve(s, width)
        cut = width == NARROW_W and any(not (s.en >> j & 1) for j in range(2, NARROW_W)) and not s.first
        out.append(Step(width, path, cut))
        if path == "fast":
            calm = calm + 1 if w < NARROW_HIT else 0
            if w >= NARROW_HIT:
                width = LANES
            elif calm >= CALM:
                width = NARROW_W
        elif path == "ambiguous":
            known = False
        else:
            width, calm = LANES, 0
    return out
