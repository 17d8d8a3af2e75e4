"""The pins of cachemap_pin restated: the range algebra of the drop-in's list (merge on pin, split on unpin,
the move of cachemap_rename, the CMB200_PIN_MAX and CMB200_PIN_RANGES refusals, the file order a load keeps),
and the sampler that passes over pinned records, on oracle/evict_model.py's TableStore.  Ranges are
(u, l_first, l_last) tuples; an address is (u, l) with l = genid << 44 | page."""
from __future__ import annotations

from oracle.evict_model import TableStore, pick, _TOMB

PNUM = 44
PIN_RANGES = 4096
TO_END = (1 << 64) - 1


def normalize(ranges) -> list:
    """Sorted by (u, l_first), with ranges of one u that overlap or touch merged."""
    out: list = []
    for u, f, l in sorted(ranges):
        if out and out[-1][0] == u and f <= out[-1][2] + 1:
            out[-1] = (u, out[-1][1], max(out[-1][2], l))
        else:
            out.append((u, f, l))
    return out


def cut(ranges, u, f, l):
    """-> (ranges without the pages of u in [f, l], the pages taken as ranges)."""
    keep, taken = [], []
    for r in ranges:
        if r[0] != u or r[2] < f or r[1] > l:
            keep.append(r)
            continue
        if r[1] < f:
            keep.append((u, r[1], f - 1))
        if r[2] > l:
            keep.append((u, l + 1, r[2]))
        taken.append((u, max(r[1], f), min(r[2], l)))
    return keep, taken


def pages(ranges) -> int:
    return sum(l - f + 1 for _, f, l in ranges)


def has(ranges, a) -> bool:
    return any(u == a[0] and f <= a[1] <= l for u, f, l in ranges)


def ranges_of(u, ls) -> list:
    """The runs of consecutive values in the sorted list ls, as ranges of u."""
    out: list = []
    for l in ls:
        if out and out[-1][2] + 1 == l:
            out[-1] = (u, out[-1][1], l)
        else:
            out.append((u, l, l))
    return out


def span(pshift, genid, off, size):
    """compose_span: the first and last l that bytes [off, off + size) of generation genid overlap, or None
    when the first page does not fit 44 bits.  The end saturates at page 2^44 - 1."""
    first = off >> pshift
    if first >> PNUM:
        return None
    end = min(off + size - 1, TO_END)
    last = min(end >> pshift, (1 << PNUM) - 1)
    return genid << PNUM | first, genid << PNUM | last


class Pins:
    """The drop-in's list for a map of `capacity` pages at page size 2^pshift, with CMB200_PIN_MAX = pin_max
    (None: the default) clamped as the drop-in clamps it."""

    def __init__(self, capacity: int, pshift: int = 12, pin_max: int | None = None):
        self.pshift = pshift
        self.max = capacity // 4 if pin_max is None else min(pin_max, capacity // 2)
        self.ranges: list = []

    def pin(self, u, genid, off, size) -> int:
        if size == 0 or size == TO_END:
            return -1
        s = span(self.pshift, genid, off, size)
        if s is None or self.max == 0:
            return -1
        nxt = normalize(self.ranges + [(u, *s)])
        if len(nxt) > PIN_RANGES or pages(nxt) > self.max:
            return -1
        added = pages(nxt) - pages(self.ranges)
        self.ranges = nxt
        return added

    def unpin(self, u, genid, off, size) -> int:
        s = span(self.pshift, genid, off, size) if size else None
        if s is None:
            return 0
        nxt, _ = cut(self.ranges, u, *s)
        if len(nxt) > PIN_RANGES:
            return 0
        removed = pages(self.ranges) - pages(nxt)
        self.ranges = nxt
        return removed

    def rename(self, frm, to, genid) -> None:
        first = genid << PNUM
        last = first | ((1 << PNUM) - 1)
        keep, _ = cut(self.ranges, to, first, last)
        keep, moved = cut(keep, frm, first, last)
        nxt = normalize(keep + [(to, f, l) for _, f, l in moved])
        if len(nxt) <= PIN_RANGES:
            self.ranges = nxt

    def load(self, file_ranges) -> None:
        """The ranges of a pins file, in file order, up to the first one that is malformed, out of order or
        over the budget."""
        self.ranges = []
        total = 0
        for r in file_ranges:
            u, f, l = r
            prev = self.ranges[-1] if self.ranges else None
            if f > l or (prev and (u < prev[0] or (u == prev[0] and f <= prev[2]))) or \
                    l - f + 1 > self.max - total or len(self.ranges) == PIN_RANGES:
                break
            self.ranges.append(r)
            total += l - f + 1


class PinnedTableStore(TableStore):
    """TableStore whose draws pass over pinned addresses: the first live, unpinned slot at or after the draw.
    When every live record is pinned no draw finds one, and the put evicts nothing."""

    def __init__(self, *args, pinned=(), **kw):
        super().__init__(*args, **kw)
        self.pinned = list(pinned)

    def _sample(self):
        i = self.draw(self.slots)
        for _ in range(self.slots):
            k = self.table[i]
            if k is not None and k is not _TOMB and not has(self.pinned, k):
                return k
            i = (i + 1) % self.slots
        return None

    def _evict(self) -> None:
        cand = [self._sample() for _ in range(3)]
        if None in cand:                            # only when every live record is pinned
            return
        victim = cand[pick(*(self.ts[c] for c in cand))]
        self.table[self.at.pop(victim)] = _TOMB
        del self.ts[victim]
        self.evicted.append(victim)
