"""Admission by frequency (CMB200_ADMIT=freq) restated, for its tests and tools/admit_bench.py.

`Sketch` is the engine's count-min sketch (cachemap_b200.h, CMB200_FREQ): 4 rows of `width` 4-bit
counters, the same index function (cmb200_freq_index), saturation at 15, and the halving that the launch
taking the count to the period enqueues.  `words()` packs it as cmb200_freq_read returns it.

`AdmitStore` and `AdmitTableStore` are oracle/evict_model.py's two samplers with the drop-in's admission
rule on top: every get counts its key in the sketch of the engine that owns it (cmb200_owner), and a put at
capacity pairs the incoming page with the victim the sampler picks; the page is stored, and the victim
evicted, only if the page's estimate is strictly greater than the victim's.  A rejected page is not stored
and its key is removed, so an older version is never served.  With admit=False they are the samplers of
evict_model, draw for draw.

The workloads address pages as the drop-in does, (nhid, page) with genid 0, so the keys, owners and sketch
indices are those of a cachemap of 4 KiB pages.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import evict_model  # noqa: E402

# cmb200_freq_index's constants (include/cachemap_b200.h), one odd multiplier per row
ROW_MUL = (0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0xD6E8FEB86659FD93)
M64 = (1 << 64) - 1


def fnv_addr(u: int, l: int) -> int:
    """The store key: FNV-1a-64 over the 16 bytes of {u, l} (filemap.c:18-24)."""
    h = 14695981039346656037
    for v in (u, l):
        for i in range(8):
            h = ((h ^ ((v >> (8 * i)) & 0xFF)) * 0x100000001B3) & M64
    return h


def freq_index(key: int, row: int, log2_width: int) -> int:
    return ((key * ROW_MUL[row]) & M64) >> (64 - log2_width)


def owner(key: int, g: int) -> int:
    return ((key >> 32) * g) >> 32


def _pow2_at_least(v: int) -> int:
    p = 1
    while p < v:
        p <<= 1
    return p


class Sketch:
    """One engine's sketch.  `launch(keys)` is one counting launch: every key +1 on its four counters, then
    a halving if the count since the last one has reached the period."""

    def __init__(self, capacity: int = 0, table_slots: int = 0):
        if capacity:
            width = _pow2_at_least(capacity)
        else:
            cap = _pow2_at_least(table_slots) if table_slots else _pow2_at_least(4 * 1024)
            width = min(max(cap, 1024), 1 << 27) // 4
        self.width = min(max(width, 16), 1 << 32)
        self.log2w = self.width.bit_length() - 1
        self.period = 10 * (capacity or self.width)
        self.c = [bytearray(self.width) for _ in range(4)]
        self.increments = self.since = self.halvings = 0

    def index(self, key: int, row: int) -> int:
        return freq_index(key, row, self.log2w)

    def add(self, key: int) -> None:
        for r in range(4):
            row, j = self.c[r], self.index(key, r)
            if row[j] < 15:
                row[j] += 1

    def halve(self) -> None:
        self.c = [bytearray((np.frombuffer(row, dtype=np.uint8) >> 1).tobytes()) for row in self.c]

    def launch(self, keys) -> None:
        keys = list(keys)
        for k in keys:
            self.add(k)
        self.increments += len(keys)
        self.since += len(keys)
        if self.since >= self.period:
            self.halve()
            self.since = 0
            self.halvings += 1

    def estimate(self, key: int) -> int:
        return min(self.c[r][self.index(key, r)] for r in range(4))

    def words(self) -> np.ndarray:
        """The sketch as cmb200_freq_read copies it: row r at words [r w/16, (r+1) w/16), counter j in the
        nibble j % 16 of word j / 16."""
        nib = np.frombuffer(b"".join(self.c), dtype=np.uint8).reshape(4, self.width // 16, 16).astype(np.uint64)
        shifts = (np.arange(16, dtype=np.uint64) * np.uint64(4))
        return (nib << shifts).sum(axis=2, dtype=np.uint64).reshape(-1)


def admits(page_estimate: int, victim_estimate: int) -> bool:
    """The drop-in's rule (filemap_admit_n): strictly more often asked for than the victim."""
    return page_estimate > victim_estimate


class _Admission:
    """Mixed into a store of evict_model: addresses are (nhid, page) pairs."""

    def _admission(self, admit: bool, engines: int, per_engine_capacity: int) -> None:
        self.admit = admit
        self.engines = engines
        self.sketches = [Sketch(per_engine_capacity) for _ in range(engines)] if admit else []
        self.admitted = self.rejected = 0

    def _sketch(self, key: int) -> Sketch:
        return self.sketches[owner(key, self.engines)]

    def estimate(self, a) -> int:
        k = fnv_addr(*a)
        return self._sketch(k).estimate(k)

    def get(self, a) -> bool:
        if self.admit:
            k = fnv_addr(*a)
            self._sketch(k).launch([k])
        return super().get(a)

    def _decide(self, a, victim) -> bool:
        """True: evict victim and store a.  False: a is rejected."""
        if admits(self.estimate(a), self.estimate(victim)):
            self.admitted += 1
            return True
        self.rejected += 1
        return False


class AdmitStore(_Admission, evict_model.Store):
    def __init__(self, capacity: int, touch: bool, admit: bool, engines: int = 1, **kw):
        evict_model.Store.__init__(self, capacity, touch, **kw)
        self._admission(admit, engines, -(-capacity // engines))

    def put(self, a) -> None:
        if not (self.admit and self.capacity and len(self.keys) >= self.capacity):
            return super().put(a)
        self.clock += 1
        cand = [self.keys[self.draw(len(self.keys))] for _ in range(3)]
        victim = cand[evict_model.pick(*(self.ts[c] for c in cand))]
        if self._decide(a, victim):
            self._remove(victim)
            self.evicted.append(victim)
            if a not in self.ts:
                self.pos[a] = len(self.keys)
                self.keys.append(a)
            self.ts[a] = self.clock
        elif a in self.ts:
            self._remove(a)


class AdmitTableStore(_Admission, evict_model.TableStore):
    def __init__(self, capacity: int, touch: bool, admit: bool, engines: int = 1, **kw):
        evict_model.TableStore.__init__(self, capacity, touch, **kw)
        self._admission(admit, engines, -(-capacity // engines))

    def put(self, a) -> None:
        if not (self.admit and self.capacity and len(self.at) >= self.capacity):
            return super().put(a)
        self.clock += 1
        cand = [self._sample() for _ in range(3)]
        victim = cand[evict_model.pick(*(self.ts[c] for c in cand))]
        if self._decide(a, victim):
            self.table[self.at.pop(victim)] = evict_model._TOMB
            del self.ts[victim]
            self.evicted.append(victim)
            if a not in self.at:
                self.at[a] = self._claim(a)
            self.ts[a] = self.clock
        elif a in self.at:
            self.table[self.at.pop(a)] = evict_model._TOMB
            del self.ts[a]


def _store(touch, admit, capacity, seed, table, engines):
    return (AdmitTableStore if table else AdmitStore)(capacity, touch, admit, engines=engines, seed=seed)


HOT_NHID, COLD_NHID = 1000, 2000


def hot_cold(touch: bool, admit: bool = False, capacity: int = 4096, hot: int = 1024, steps: int = 65536,
             warmup: int = 16384, seed: int = 0, table: bool = False, engines: int = 1) -> float:
    """evict_model.hot_cold with admission: hot page (step mod hot), put on a miss, then one cold page put."""
    s = _store(touch, admit, capacity, seed, table, engines)
    hits = reads = 0
    for t in range(steps):
        h = (HOT_NHID, t % hot)
        hit = s.get(h)
        if not hit:
            s.put(h)
        s.put((COLD_NHID, t))
        if t >= warmup:
            reads += 1
            hits += hit
    return hits / reads


def scan(touch: bool, admit: bool = False, capacity: int = 4096, hot: int = 2048, per_read: int = 1,
         steps: int = 65536, warmup: int = 16384, seed: int = 0, table: bool = False, engines: int = 1) -> float:
    """A hot set read at random while a scan goes by: each step gets a uniformly drawn hot page (put on a
    miss), then `per_read` scan pages that are never read again, each missed and put, as a backup or a
    grep -r reads through the mount.  Returns the hot set's hit ratio after `warmup` steps."""
    s = _store(touch, admit, capacity, seed, table, engines)
    rng = random.Random(seed ^ 0x5CA7)
    hits = reads = 0
    nxt = 0
    for t in range(steps):
        h = (HOT_NHID, rng.randrange(hot))
        hit = s.get(h)
        if not hit:
            s.put(h)
        for _ in range(per_read):
            c = (COLD_NHID, nxt)
            nxt += 1
            if not s.get(c):
                s.put(c)
        if t >= warmup:
            reads += 1
            hits += hit
    return hits / reads
