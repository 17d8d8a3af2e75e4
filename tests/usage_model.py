"""A restatement of cachemap_residency and cachemap_usage over a set of records.

records: {(u, l): (record length, in the host tier, ts)}, where l = genid << 44 | page and a record's length
is its 24-byte prefix plus its LZ4 block or raw page; pins: sorted, disjoint ranges (u, l_first, l_last) as
tests/pin_model.py keeps them.  Rows are tuples in USAGE_DTYPE's field order:
(nhid, genid, 0, pages, tier_pages, pinned_pages, stored_bytes, first_page, last_page, oldest_ts, newest_ts).
"""
import numpy as np

PNUM = 44
PAGE_MASK = (1 << PNUM) - 1
TO_END = (1 << 64) - 1
PREFIX = 24
IN_HBM, IN_TIER, PINNED = 1, 2, 4
FIELDS = ("nhid", "genid", "reserved", "pages", "tier_pages", "pinned_pages", "stored_bytes", "first_page",
          "last_page", "oldest_ts", "newest_ts")


def record_len(clen: int, bsize: int) -> int:
    """The stored length of a record whose LZ4 block is clen bytes (0: the page is stored raw)."""
    return PREFIX + (clen or bsize)


def span(pshift, genid, off, size):
    """The first and last l of the pages that bytes [off, off + size) overlap, partial pages at both ends
    included; None when cachemap_residency refuses: size 0 or TO_END, an end past 2^64, or a first or last
    page that does not fit 44 bits."""
    if size == 0 or size == TO_END or off + size - 1 > TO_END:
        return None
    first, last = off >> pshift, (off + size - 1) >> pshift
    if first >> PNUM or last >> PNUM:
        return None
    return genid << PNUM | first, genid << PNUM | last


def pinned(pins, u, l) -> bool:
    return any(pu == u and f <= l <= t for pu, f, t in pins)


def engine_residency(records, u, l_first, l_last) -> np.ndarray:
    """cmb200_residency into a zeroed vector: 1 = arena, 2 = host tier."""
    out = np.zeros(l_last - l_first + 1, dtype=np.uint8)
    for (ru, rl), (_, tier, _) in records.items():
        if ru == u and l_first <= rl <= l_last:
            out[rl - l_first] = 2 if tier else 1
    return out


def residency(records, pins, pshift, u, genid, off, size):
    """-> (pages cached, vector), or (-1, None) when refused."""
    s = span(pshift, genid, off, size)
    if s is None:
        return -1, None
    vec = engine_residency(records, u, *s)
    cached = int(np.count_nonzero(vec))
    for pu, f, t in pins:
        if pu == u and t >= s[0] and f <= s[1]:
            vec[max(f, s[0]) - s[0]:min(t, s[1]) - s[0] + 1] |= PINNED
    return cached, vec


def rows(records, pins) -> list:
    """One row per object (u, genid) with a record, in no particular order."""
    acc = {}
    for (u, l), (length, tier, ts) in records.items():
        k = (u, l >> PNUM)
        page = l & PAGE_MASK
        pin = pinned(pins, u, l)
        r = acc.get(k)
        if r is None:
            acc[k] = [u, l >> PNUM, 0, 1, int(tier), int(pin), length, page, page, ts, ts]
        else:
            r[3] += 1; r[4] += int(tier); r[5] += int(pin); r[6] += length
            r[7] = min(r[7], page); r[8] = max(r[8], page); r[9] = min(r[9], ts); r[10] = max(r[10], ts)
    return [tuple(r) for r in acc.values()]


def order(rs) -> list:
    """The public order: stored_bytes descending, then nhid ascending, then genid ascending."""
    return sorted(rs, key=lambda r: (-r[6], r[0], r[1]))


def usage(records, pins, max_rows):
    """-> (objects, the first min(max_rows, objects) rows in the public order)."""
    rs = order(rows(records, pins))
    return len(rs), rs[:max_rows]


def merge(row_lists) -> list:
    """Rows of one object found on several engines, summed into one row (the order is not applied)."""
    acc = {}
    for rs in row_lists:
        for r in rs:
            k = (r[0], r[1])
            a = acc.get(k)
            if a is None:
                acc[k] = list(r)
            else:
                for i in (3, 4, 5, 6):
                    a[i] += r[i]
                a[7] = min(a[7], r[7]); a[8] = max(a[8], r[8]); a[9] = min(a[9], r[9]); a[10] = max(a[10], r[10])
    return [tuple(a) for a in acc.values()]


def as_tuples(arr) -> list:
    """A USAGE_DTYPE array (edge_fuse_b200.binding) as row tuples."""
    return [tuple(int(x[f]) for f in FIELDS) for x in arr]
