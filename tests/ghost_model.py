"""Ghost entries (CMB200_GHOST) restated, for their tests and tools/ghost_bench.py.

`GhostTable` is one engine's ghost table (include/cachemap_b200.h): `entries` 32-byte entries {u, l, stamp, 0}
in 4-way sets, the set of an address from cmb200_ghost_set of its store key, the eviction clock, the insert
rule (the live ghost of the same address, else the first empty way, else the oldest stamp), consumption by
probes with the refault distance d = clock - stamp (the evictions after it) in 64 buckets of entries / 64,
and removal.  A cleared entry keeps its address and only its stamp goes to 0, as on the GPU, so `words()` equals cmb200_ghost_read
word for word.

`GhostStore` and `GhostTableStore` are oracle/evict_model.py's two samplers with one ghost table: every victim
is evicted by one call (one stamp), and every get that misses probes.  `GhostTable.would_hit(extra)` is what
cachemap_hit_curve answers: the refaults whose distance lies below `extra` rounded down to a bucket.

The workloads address pages as the drop-in does, (nhid, page) with genid 0.
"""
from __future__ import annotations

import bisect
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import evict_model  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from admit_model import HOT_NHID, COLD_NHID, fnv_addr, _pow2_at_least  # noqa: E402

GHOST_MUL = 0x9FB21C651E98DF25       # cmb200_ghost_set's multiplier (include/cachemap_b200.h)
M64 = (1 << 64) - 1
ZIPF_NHID = 3000


def ghost_set(key: int, log2_sets: int) -> int:
    return ((key * GHOST_MUL) & M64) >> (64 - log2_sets)


def table_entries(capacity: int = 0, table_slots: int = 0) -> int:
    """The engine's sizing: the power of two at or above capacity (table_slots / 4 without one), >= 256."""
    if capacity:
        n = _pow2_at_least(capacity)
    else:
        cap = _pow2_at_least(table_slots) if table_slots else _pow2_at_least(4 * 1024)
        n = min(max(cap, 1024), 1 << 27) // 4
    return min(max(n, 256), 1 << 32)


class GhostTable:
    def __init__(self, capacity: int = 0, table_slots: int = 0):
        self.entries = table_entries(capacity, table_slots)
        self.log2_sets = (self.entries // 4).bit_length() - 1
        self.width = self.entries // 64
        self.tab = [[0, 0, 0] for _ in range(self.entries)]     # u, l, stamp
        self.clock = 0
        self.inserted = self.replaced = self.removed = 0
        self.probes = self.refaults = self.beyond = 0
        self.hist = [0] * 64
        self.distances: list = []                                 # every refault's d, in order

    def _ways(self, a):
        s = ghost_set(fnv_addr(*a), self.log2_sets)
        return self.tab[4 * s: 4 * s + 4]

    def _take(self, a) -> int:
        for w in self._ways(a):
            if (w[0], w[1]) == tuple(a) and w[2]:
                s, w[2] = w[2], 0
                return s
        return 0

    def insert(self, addrs) -> None:
        """One evicting call: its removed addresses in order, stamped clock + 1, clock + 2, ..."""
        for a in addrs:
            self.clock += 1
            ways = self._ways(a)
            pick = next((w for w in ways if w[2] and (w[0], w[1]) == tuple(a)), None)
            if pick is None:
                pick = next((w for w in ways if not w[2]), None)
            if pick is None:
                pick = min(ways, key=lambda w: w[2])
                self.replaced += 1
            pick[0], pick[1], pick[2] = a[0], a[1], self.clock
            self.inserted += 1

    def probe(self, addrs) -> None:
        """One get call's misses, in request order."""
        for a in addrs:
            self.probes += 1
            s = self._take(a)
            if not s:
                continue
            self.refaults += 1
            d = self.clock - s
            self.distances.append(d)
            if d >= self.entries:
                self.beyond += 1
            else:
                self.hist[d // self.width] += 1

    def remove(self, addrs) -> None:
        for a in addrs:
            self.removed += self._take(a) != 0

    def remove_span(self, u: int, l_first: int, l_last: int) -> None:
        for w in self.tab:
            if w[0] == u and l_first <= w[1] <= l_last and w[2]:
                w[2] = 0
                self.removed += 1

    def would_hit(self, extra: int) -> int:
        """cachemap_hit_curve for one engine: the refaults of the buckets wholly below `extra`."""
        return sum(self.hist[:min(64, extra // self.width)])

    def words(self) -> np.ndarray:
        out = np.zeros((self.entries, 4), dtype=np.uint64)
        out[:, :3] = np.array(self.tab, dtype=np.uint64)
        return out

    def stats(self) -> dict:
        return dict(entries=self.entries, bucket_width=self.width, clock=self.clock, inserted=self.inserted,
                    replaced=self.replaced, removed=self.removed, probes=self.probes, refaults=self.refaults,
                    beyond=self.beyond, hist=list(self.hist))


class _Ghosts:
    """Mixed into a store of evict_model: evictions leave ghosts, misses probe them."""

    def _ghosts(self, capacity: int) -> None:
        self.ghosts = GhostTable(capacity)

    def get(self, a) -> bool:
        hit = super().get(a)
        if not hit:
            self.ghosts.probe([a])
        return hit

    def _evict(self) -> None:
        n = len(self.evicted)
        super()._evict()
        self.ghosts.insert(self.evicted[n:])


class GhostStore(_Ghosts, evict_model.Store):
    def __init__(self, capacity: int, touch: bool, **kw):
        evict_model.Store.__init__(self, capacity, touch, **kw)
        self._ghosts(capacity)


class GhostTableStore(_Ghosts, evict_model.TableStore):
    def __init__(self, capacity: int, touch: bool, **kw):
        evict_model.TableStore.__init__(self, capacity, touch, **kw)
        self._ghosts(capacity)


def _reads(workload: str, steps: int, seed: int, hot: int, keys: int, alpha: float):
    """The workload's accesses: (address, read) pairs.  read: a get (put on a miss); else a put only."""
    rng = random.Random(seed ^ 0x9057)
    if workload == "hot_cold":
        for t in range(steps):
            yield (HOT_NHID, t % hot), True
            yield (COLD_NHID, t), False
    elif workload == "scan":
        for t in range(steps):
            yield (HOT_NHID, rng.randrange(hot)), True
            yield (COLD_NHID, t), True
    elif workload == "zipf":
        w = np.arange(1, keys + 1, dtype=np.float64) ** -alpha
        cdf = list(np.cumsum(w / w.sum()))
        for _ in range(steps):
            yield (ZIPF_NHID, min(bisect.bisect_left(cdf, rng.random()), keys - 1)), True
    else:
        raise ValueError(workload)


def run(workload: str, touch: bool, capacity: int, steps: int = 32768, warmup: int = 8192, seed: int = 0,
        table: bool = True, hot: int = 1024, keys: int = 30000, alpha: float = 0.9, extra=()):
    """One run at `capacity`.  Returns (hit ratio of the gets after warmup, {extra: predicted hit ratio}).
    The prediction counts the refaults of the measured gets, as cachemap_hit_curve counts the misses since
    create, so it adds to the measured hits exactly the misses that the curve says a larger store serves."""
    s = (GhostTableStore if table else GhostStore)(capacity, touch, seed=seed)
    hits = reads = 0
    hist0 = None
    for t, (a, read) in enumerate(_reads(workload, steps, seed, hot, keys, alpha)):
        if t == warmup * (2 if workload in ("hot_cold", "scan") else 1):
            hist0 = list(s.ghosts.hist)
        counted = hist0 is not None
        if read:
            hit = s.get(a)
            if counted:
                reads += 1
                hits += hit
            if hit:
                continue
        s.put(a)
    g = s.ghosts
    pred = {}
    for x in extra:
        b = min(64, x // g.width)
        pred[x] = (hits + sum(g.hist[:b]) - sum(hist0[:b])) / reads
    return hits / reads, pred
