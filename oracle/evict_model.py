"""The store's eviction policy restated on a logical clock, for the tests of CMB200_EVICT=access.

Before every put at capacity the reference retires the oldest of three records drawn at random
(cachemap.c:17-48); the drop-in does the same with the timestamps cmb200_sample reports.  What the
timestamp means is the policy: the put time ("put", the reference's), or the last hit as well
("access", CMB200_TOUCH).  The clock here counts operations, so the model says what the policy does
to a workload, not how fast.  `pick` is the reference's comparison, ties included.

Two samplers.  `Store` draws uniformly over the live records.  `TableStore` draws as the store does
(k_sample, the policy-equivalent of filemap_get_rand): the records sit in a linear-probing table of
4 x capacity slots, a removed record leaves a tombstone that a later claim of its chain reuses (the table
is rebuilt only by compaction, which a store of small records seldom needs), and a draw is the first live
slot at or after a uniform one.  A record behind a long run of empty and dead slots is drawn more often
than one right behind another record; that changes what the policies keep, "access" more than "put".
"""
from __future__ import annotations

import random


def pick(a: int, b: int, c: int) -> int:
    """Index (0, 1, 2) of the victim among three sampled timestamps, as cachemap.c:29-41 chooses it."""
    if a < b:
        return 2 if a > c else 0
    return 2 if b > c else 1


class Store:
    """Records keyed by address, each with a timestamp; `draw(n)` gives an index in [0, n)."""

    def __init__(self, capacity: int, touch: bool, draw=None, seed: int = 0):
        self.capacity = capacity
        self.touch = touch
        self.clock = 0
        self.ts: dict = {}
        self.keys: list = []            # live addresses, for uniform draws
        self.pos: dict = {}
        rng = random.Random(seed)
        self.draw = draw if draw is not None else (lambda n: rng.randrange(n))
        self.evicted: list = []

    def __len__(self) -> int:
        return len(self.keys)

    def get(self, a) -> bool:
        self.clock += 1
        if a not in self.ts:
            return False
        if self.touch:
            self.ts[a] = self.clock
        return True

    def put(self, a) -> None:
        self.clock += 1
        if self.capacity and len(self.keys) >= self.capacity:
            self._evict()
        if a not in self.ts:
            self.pos[a] = len(self.keys)
            self.keys.append(a)
        self.ts[a] = self.clock

    def _evict(self) -> None:
        cand = [self.keys[self.draw(len(self.keys))] for _ in range(3)]
        victim = cand[pick(*(self.ts[c] for c in cand))]
        self._remove(victim)
        self.evicted.append(victim)

    def _remove(self, a) -> None:
        i = self.pos.pop(a)
        last = self.keys.pop()
        if last != a:
            self.keys[i] = last
            self.pos[last] = i
        del self.ts[a]


_TOMB = object()


class TableStore(Store):
    """Store whose draws are k_sample's over a table of `slots` slots (4 x capacity by default).  `home(a)`
    gives an address's home slot (default: a seeded random slot per address)."""

    def __init__(self, capacity: int, touch: bool, draw=None, seed: int = 0, slots: int = 0, home=None):
        super().__init__(capacity, touch, draw, seed)
        self.slots = slots or 4 * capacity
        self.table: list = [None] * self.slots      # None = empty, _TOMB = dead, else the address
        self.at: dict = {}
        homes: dict = {}
        rng = random.Random(seed ^ 0x5EED)
        self.home = home if home is not None else (lambda a: homes.setdefault(a, rng.randrange(self.slots)))

    def __len__(self) -> int:
        return len(self.at)

    def put(self, a) -> None:
        self.clock += 1
        if self.capacity and len(self.at) >= self.capacity:
            self._evict()
        if a not in self.at:
            self.at[a] = self._claim(a)
        self.ts[a] = self.clock

    def _claim(self, a) -> int:
        """table_find_or_claim: the first tombstone of the chain once the chain ends in an empty slot."""
        i, tomb = self.home(a), None
        for _ in range(self.slots):
            k = self.table[i]
            if k is None:
                j = i if tomb is None else tomb
                self.table[j] = a
                return j
            if k is _TOMB and tomb is None:
                tomb = i
            i = (i + 1) % self.slots
        assert tomb is not None, "table full"
        self.table[tomb] = a
        return tomb

    def _sample(self):
        i = self.draw(self.slots)
        for _ in range(self.slots):
            k = self.table[i]
            if k is not None and k is not _TOMB:
                return k
            i = (i + 1) % self.slots
        raise AssertionError("empty table")

    def _evict(self) -> None:
        cand = [self._sample() for _ in range(3)]
        victim = cand[pick(*(self.ts[c] for c in cand))]
        self.table[self.at.pop(victim)] = _TOMB
        del self.ts[victim]
        self.evicted.append(victim)


def hot_cold(touch: bool, capacity: int = 4096, hot: int = 1024, steps: int = 65536, warmup: int = 16384,
             seed: int = 0, table: bool = False) -> float:
    """The hot and cold workload: each step gets hot page (step mod hot) and puts it on a miss, as edgefs
    reads a page (edgefs.c:1179-1195), then puts one cold page that is never read.  Returns the hot set's
    hit ratio over the steps after `warmup`.  table: draw as the store does (TableStore)."""
    s = (TableStore if table else Store)(capacity, touch, seed=seed)
    hits = reads = 0
    for t in range(steps):
        h = ("h", t % hot)
        hit = s.get(h)
        if not hit:
            s.put(h)
        s.put(("c", t))
        if t >= warmup:
            reads += 1
            hits += hit
    return hits / reads
