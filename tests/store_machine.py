"""A stateful model of one engine and a seeded generator of operation logs that drive it.

The model (`Model`) wraps oracle StoreModel, which decides hit, miss and bad entry and holds each key's
exact record bytes, and adds what the engine's bookkeeping must agree with: each record's page, tier
(arena or host), ring position in the host tier, fingerprint, parse checkpoints and timestamp, the arena's
bump pointer and the host tier's ring.  `gen_ops` turns a seed into a replayable list of operations over
every engine call; `census` runs a log through the model alone and reports which rare events it reaches.
CPU only: the GPU test (test_gpu_store_machine.py) drives an engine and this model side by side.
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass, field

import numpy as np

import datagen
import key_edges
from ckpt_def import ckpt_words

FINGERPRINT, VERIFY, TOUCH = 1, 2, 4
MISS, HIT, INVALID, BAD_ENTRY = 0, 1, 2, 3
KEY_SENTINELS = (0, (1 << 64) - 1)


@dataclass(frozen=True)
class MachineConfig:
    name: str
    pshift: int
    accel: int
    flags: int
    tier_bytes: int            # 0: no host tier
    table_slots: int
    arena_bytes: int
    load_slots: int            # geometry of the engine a snapshot is loaded into
    load_arena: int
    env: tuple                 # ((variable, value), ...) set before the engine is created
    us: tuple                  # object ids (u) of the key universe
    nl: int                    # pages per object: l in [0, nl)
    batch: int                 # largest put batch
    steps: int
    seeds: tuple
    exact_head: bool           # no per-warp arena segments: the model tracks the bump pointer exactly
    events: tuple              # the census events every configuration's seeds must reach
    max_batch: int = 256

    @property
    def bsize(self) -> int:
        return 1 << self.pshift

    @property
    def cap(self) -> int:
        return self.table_slots

    def environ(self) -> dict:
        return dict(self.env)


ALL_EVENTS = ("drop", "compact", "rebuild", "wrap", "inval_keyed", "inval_scan", "load", "promote_after_demote_after_compact")

CONFIGS = {
    "A": MachineConfig("A", 12, 12, VERIFY, 96 << 10, 1024, 512 << 10, 2048, 2 << 20,
                       (("CMB200_SEG_KB", "0"),), (3, 5, 7), 80, 48, 70, (11, 12), True, ALL_EVENTS),
    "B": MachineConfig("B", 16, 12, FINGERPRINT | TOUCH, 0, 1024, 512 << 20, 4096, 384 << 20,
                       (("CMB200_SEG_KB", "512"),), (3, 5), 24, 12, 30, (21, 22), False,
                       ("compact", "rebuild", "inval_keyed", "inval_scan", "load")),
    "C": MachineConfig("C", 17, 12, VERIFY, 1 << 20, 1024, 3 << 20, 2048, 12 << 20,
                       (), (3, 5), 16, 8, 30, (31, 32), True,
                       ("drop", "compact", "rebuild", "wrap", "inval_keyed", "inval_scan", "load",
                        "promote_after_demote_after_compact")),
    "D": MachineConfig("D", 12, 0, 0, 0, 1024, 1536 << 10, 2048, 4 << 20,
                       (("CMB200_CKPT", "0"),), (3, 5, 7), 80, 48, 60, (41, 42), True,
                       ("drop", "compact", "rebuild", "inval_keyed", "inval_scan", "load")),
}


def edge_addrs() -> list:
    """Addresses that share a store key with another one, and addresses of the table's sentinel keys."""
    fx = key_edges.load()
    return [a for g in fx["groups"].values() for a in g]


PURGE_U = 99


def purge_addrs(cfg: MachineConfig) -> list:
    """Keys put once and deleted together: more tombstones than cap / 8 whatever the universe's size."""
    return [(PURGE_U, l) for l in range(cfg.table_slots // 8 + 24)]


def universe(cfg: MachineConfig) -> list:
    return [(u, l) for u in cfg.us for l in range(cfg.nl)] + edge_addrs() + purge_addrs(cfg)


def alloc(payload: int) -> int:
    return (24 + payload + 15) & ~15


# ---- model ----------------------------------------------------------------------------------------

@dataclass
class Rec:
    addr: tuple
    page: bytes
    clen: int                  # 0: raw page
    block: bytes
    ts_lo: int                 # the record's ts lies in [ts_lo, ts_hi] (equal unless a touch moved it)
    ts_hi: int
    has_fp: bool
    fp: tuple | None
    ckpt: list | None          # words of a compressed block whose chain fits, else None
    host_pos: int | None = None    # ring log position while in the host tier

    @property
    def need(self) -> int:
        return alloc(self.clen or len(self.page))


@dataclass
class Counters:
    dropped: int = 0
    requests: int = 0
    hits: int = 0
    verified: int = 0
    unverified: int = 0
    retired: int = 0


class Model:
    def __init__(self, cfg: MachineConfig, oracle):
        self.cfg, self.O = cfg, oracle
        self.sm = oracle.StoreModel(cfg.pshift, cfg.accel)
        self.rec: dict[int, Rec] = {}
        self.ctr = Counters()
        self.head = 0                                  # arena bump pointer (exact_head configs)
        self.arena_size = cfg.arena_bytes
        self.cap = cfg.table_slots
        self.tier_head = 0
        self.tier_log: deque = deque()                 # [position, need, key] oldest first
        self.tomb_lo = self.tomb_hi = 0                # bounds of the table's tombstone count
        self.saturated = False                         # a drop pushed the bump pointer past the arena
        self._enc: dict = {}

    # the record a put of `page` at {u, l} makes
    def make(self, a, page: np.ndarray, ts: int) -> Rec:
        off, nh, gen = key_edges.cachemap_args(a[0], a[1], self.cfg.pshift)
        m = self.O.StoreModel(self.cfg.pshift, self.cfg.accel)
        m.put(off, nh, gen, page)
        (_, clen, payload), = m.rec.values()
        h = (page.tobytes(), self.cfg.accel)
        if h not in self._enc:
            fp = self.O.fingerprint128(page) if self.cfg.flags & (FINGERPRINT | VERIFY) else None
            ck = ckpt_words(payload, self.cfg.bsize) if clen else None
            self._enc[h] = (fp, ck)
        fp, ck = self._enc[h]
        return Rec(a, page.tobytes(), clen, payload, ts, ts, fp is not None, fp, ck)

    def key(self, a) -> int:
        return self.O.addr_key(a[0], a[1])

    def _install(self, r: Rec):
        k = self.key(r.addr)
        self.rec[k] = r
        self.sm.rec[k] = (r.addr, r.clen, r.block)

    def _remove(self, k: int, tomb: bool = True):
        self.rec.pop(k, None)
        self.sm.rec.pop(k, None)
        if tomb and k not in KEY_SENTINELS:
            self.tomb_lo += 1
            self.tomb_hi += 1

    def live(self, a):
        r = self.rec.get(self.key(a))
        return r if r is not None and r.addr == tuple(a) else None

    # put: which rows are applied (the last valid row of each key), in index order
    def put_rows(self, addrs, valid):
        last = {}
        for i, a in enumerate(addrs):
            if valid is None or valid[i]:
                last[self.key(a)] = i
        return sorted(last.values())

    def put(self, addrs, pages, ts, valid, dropped_rows):
        """Applies a put whose rows `dropped_rows` (a set of row indices) the arena dropped."""
        rows = self.put_rows(addrs, valid)
        claims = sum(1 for i in rows if self.key(addrs[i]) not in self.rec)
        self.tomb_lo = max(0, self.tomb_lo - claims)
        for i in rows:
            r = self.make(addrs[i], pages[i], int(ts[i]) if ts is not None else 0)
            self.head += r.need
            if i in dropped_rows:
                self.ctr.dropped += 1
                continue
            self._install(r)
        if dropped_rows:
            self.saturated = True

    def stand_in_drops(self, addrs, pages, valid) -> set:
        """Rows a sequential bump allocator drops (no GPU): once one allocation fails every later one
        does, since the pointer is never rolled back.  Which rows the engine drops depends on its chunk
        order; whether it drops any does not."""
        if not self.cfg.exact_head:
            return set()
        head, out = self.head, set()
        for i in self.put_rows(addrs, valid):
            n = self.make(addrs[i], pages[i], 0).need
            if head + n > self.arena_size:
                out.add(i)
            head += n
        return out

    def certain_drop(self, addrs, pages, valid) -> bool:
        return bool(self.stand_in_drops(addrs, pages, valid))

    def get(self, addrs, valid, t0=None, t1=None):
        """-> list of (status, page bytes or None); books requests, hits, verification and touches."""
        out = []
        for i, a in enumerate(addrs):
            if valid is not None and not valid[i]:
                out.append((INVALID, None))
                continue
            off, nh, gen = key_edges.cachemap_args(a[0], a[1], self.cfg.pshift)
            st, pg = self.sm.get_status(off, nh, gen)
            self.ctr.requests += 1
            if st == "hit":
                self.ctr.hits += 1
                r = self.rec[self.key(a)]
                assert pg == r.page
                if self.cfg.flags & VERIFY:
                    if r.has_fp:
                        self.ctr.verified += 1
                    else:
                        self.ctr.unverified += 1
                if self.cfg.flags & TOUCH and t0 is not None:
                    r.ts_lo = max(r.ts_lo, t0)
                    r.ts_hi = max(r.ts_hi, t1)
                out.append((HIT, pg))
            else:
                out.append((BAD_ENTRY if st == "bad entry" else MISS, None))
        return out

    def unset(self, addrs):
        for a in addrs:
            k = self.key(a)
            if k in self.rec:
                self._remove(k)

    def invalidate(self, u, lf, ll) -> int:
        gone = [k for k, r in self.rec.items() if r.addr[0] == u and lf <= r.addr[1] <= ll]
        for k in gone:
            self._remove(k)
        return len(gone)

    def rebuild_check(self):
        """After an invalidate or a compaction: the table is rebuilt when tombstones > cap / 8.
        -> True (certain), False (certainly not) or None (the bounds do not decide)."""
        lim = self.cap // 8
        if self.tomb_lo > lim:
            self.tomb_lo = self.tomb_hi = 0
            return True
        if self.tomb_hi <= lim:
            return False
        self.tomb_lo = 0
        return None

    def compact(self):
        self.head = sum(r.need for r in self.rec.values() if r.host_pos is None)
        self.saturated = False

    # host tier: a ring in demotion order (engine.cu demote_records / demote_group)
    def demote(self, addrs) -> tuple[int, list]:
        """-> (records moved, keys a wrap retired)."""
        size = self.cfg.tier_bytes
        moved, seen = [], set()
        for a in addrs:
            r = self.live(a)
            if r is None or r.host_pos is not None or id(r) in seen:
                continue
            seen.add(id(r))
            moved.append(r)
        # groups as demote_records forms them: one bounce buffer (at most one lap) and max_batch records
        # each; a group first retires what its region overwrites, then publishes its records
        cap = min(size, min(self.cfg.max_batch, 4096) * self.cfg.bsize)
        retired, k, pos = [], 0, self.tier_head
        while k < len(moved):
            start, grp = pos, []
            while k < len(moved) and len(grp) < self.cfg.max_batch:
                need, p = moved[k].need, pos
                if p % size + need > size:
                    p += size - p % size                         # no record straddles the end of the ring
                if p + need - start > cap:
                    break
                grp.append((moved[k], p))
                pos = p + need
                k += 1
            while self.tier_log and self.tier_log[0][0] + size < pos:
                p, need, key = self.tier_log.popleft()
                r = self.rec.get(key)
                if r is not None and r.host_pos == p:
                    retired.append(key)
                    self._remove(key)
                    self.ctr.retired += 1
            for r, p in grp:
                r.host_pos = p
                self.tier_log.append((p, r.need, self.key(r.addr)))
        self.tier_head = pos
        return len(moved), retired

    def promote(self, addrs) -> int:
        done, seen = 0, set()
        for a in addrs:
            r = self.live(a)
            if r is None or r.host_pos is None or id(r) in seen:
                continue
            seen.add(id(r))
            if self.head + r.need > self.arena_size:
                break
            self.head += r.need
            r.host_pos = None
            done += 1
        return done

    def load(self, cfg_slots: int, arena: int):
        """The store saved and loaded into a fresh engine: every record in its arena."""
        for r in self.rec.values():
            r.host_pos = None
        self.tier_log.clear()
        self.tier_head = 0
        self.cap, self.arena_size = cfg_slots, arena
        self.head = sum(r.need for r in self.rec.values())
        self.saturated = False
        self.tomb_lo = self.tomb_hi = 0
        self.ctr = Counters()

    # identities
    def arena_alloc(self) -> int:
        return sum(r.need for r in self.rec.values() if r.host_pos is None)

    def tier_records(self) -> int:
        return sum(1 for r in self.rec.values() if r.host_pos is not None)

    def tier_used(self) -> int:
        return self.tier_head - self.tier_log[0][0] if self.tier_log else 0

    def tier_garbage(self) -> int:
        g = 0
        for p, need, k in self.tier_log:
            r = self.rec.get(k)
            if r is None or r.host_pos != p:
                g += need
        return g

    def fp_records(self) -> int:
        return sum(1 for r in self.rec.values() if r.has_fp)


# ---- operation generator --------------------------------------------------------------------------

KINDS = "RTZMPAX"


class _Rng:
    """splitmix64 draws (datagen.words), so that a log does not depend on numpy's generators."""

    def __init__(self, seed: int):
        self.seed, self.i, self.buf = seed, 0, []

    def next(self) -> int:
        if not self.buf:
            self.buf = [int(x) for x in datagen.words(self.seed * 1_000_003 + self.i, 64)]
            self.i += 64
        return self.buf.pop()

    def below(self, n: int) -> int:
        return self.next() % n

    def chance(self, p: float) -> bool:
        return self.next() % 1_000_000 < int(p * 1_000_000)


def gen_ops(cfg: MachineConfig, seed: int) -> list:
    """A deterministic log of operations: tuples (kind, args...) with everything needed to replay them.
    A skeleton of phases reaches the rare events (overflow, compaction, tier wrap, table rebuild, load);
    the mix around it is drawn from the seed."""
    R = _Rng(seed)
    main = [(u, l) for u in cfg.us for l in range(cfg.nl)]
    edges = edge_addrs()
    ops = []
    pseq = [seed * 100_000]

    def page_spec():
        pseq[0] += 1
        k = R.below(10)
        kind = "R" if k < 2 else ("Z" if k == 2 else KINDS[R.below(len(KINDS))])
        return (kind, pseq[0])

    def pick(n, pool=None):
        pool = pool or main
        hot = pool[: max(4, len(pool) // 4)]                         # overwrite-heavy: a hot quarter
        return [hot[R.below(len(hot))] if R.chance(0.5) else pool[R.below(len(pool))] for _ in range(n)]

    def put(n=None, heavy=None, rows=None):
        n = n or 1 + R.below(cfg.batch)
        addrs = list(rows or pick(n))
        if not rows and n > 2 and R.chance(0.3):                    # duplicates in one batch
            addrs[R.below(n)] = addrs[R.below(n)]
        if R.chance(0.3):
            addrs += [edges[R.below(len(edges))] for _ in range(1 + R.below(3))]
        n = len(addrs)
        specs = [(heavy, pseq[0] + i + 1) if heavy else page_spec() for i in range(n)]
        if heavy:
            pseq[0] += n
        valid = None if R.chance(0.6) else [0 if R.chance(0.1) else 1 for _ in range(n)]
        ts = None if R.chance(0.3) else [1 + R.below(1 << 40) for _ in range(n)]
        kind = "put_async" if R.chance(0.3) else "put"
        ops.append((kind, addrs, specs, ts, valid))

    def get():
        n = 1 + R.below(min(48, 2 * cfg.batch))
        addrs = pick(n) + [edges[R.below(len(edges))] for _ in range(R.below(4))]
        small = R.chance(0.5)
        valid = None if small or R.chance(0.5) else [0 if R.chance(0.15) else 1 for _ in addrs]
        ops.append(("get_small" if small else "get", addrs, valid))

    def unset():
        addrs = pick(1 + R.below(8), main + edges)
        addrs += [addrs[0]] if R.chance(0.5) else []                # the same key twice in one batch
        ops.append(("unset", addrs))

    def invalidate(scan=None):
        keyed_max = (cfg.table_slots + 2) // 64
        scan = R.chance(0.5) if scan is None else scan
        w = keyed_max + R.below(cfg.nl) if scan else R.below(keyed_max)
        lf = R.below(cfg.nl)
        ops.append(("invalidate", cfg.us[R.below(len(cfg.us))], lf, lf + w))

    def demote(n=None):
        if cfg.tier_bytes:
            ops.append(("demote", pick(n or 1 + R.below(cfg.batch))))

    def promote():
        if cfg.tier_bytes:
            ops.append(("promote", pick(1 + R.below(cfg.batch))))

    def mix(k):
        for _ in range(k):
            x = R.below(100)
            if x < 38:
                put()
            elif x < 60:
                get()
            elif x < 68:
                unset()
            elif x < 74:
                invalidate()
            elif x < 80:
                ops.append(("sample", [R.next() for _ in range(16)]))
            elif x < 86:
                demote()
            elif x < 91:
                promote()
            elif x < 94:
                ops.append(("compact",))
            elif cfg.flags & VERIFY:
                ops.append(("verify_store",))
            else:
                get()

    # fill, then overflow the arena with incompressible pages
    for at in range(0, len(main), cfg.batch):
        put(rows=main[at:at + cfg.batch])
    mix(cfg.steps // 6)
    if cfg.exact_head:
        for _ in range(3):
            put(n=cfg.batch, heavy="R")
    mix(cfg.steps // 6)
    # compaction, then demotion (enough to wrap the ring), promotion
    ops.append(("compact",))
    if cfg.tier_bytes:
        demote(cfg.batch)
        demote(cfg.batch)
        promote()
        ops.append(("promote", list(main)))
        demote(cfg.batch)
    mix(cfg.steps // 6)
    # purge: more tombstones than cap / 8, then an invalidation (rebuild), both invalidation paths
    purge = purge_addrs(cfg)
    ops.append(("unset", main[: len(main) // 2]))
    ops.append(("compact",))
    for at in range(0, len(purge), cfg.batch):
        put(rows=purge[at:at + cfg.batch], heavy="Z")
    ops.append(("unset", purge))
    invalidate(scan=False)
    invalidate(scan=True)
    mix(cfg.steps // 6)
    ops.append(("load",))
    mix(cfg.steps // 6)
    ops.append(("compact",))
    mix(cfg.steps - 5 * (cfg.steps // 6))
    return ops


def pages_of(cfg: MachineConfig, specs) -> np.ndarray:
    return np.stack([datagen.make_page(k, cfg.bsize, s) for k, s in specs])


def describe(op) -> str:
    """One line per operation for a failure's op log."""
    k = op[0]
    if k in ("put", "put_async"):
        return f"{k} n={len(op[1])} addrs={op[1][:4]}... pages={op[2][:4]}... ts={'set' if op[3] else None} valid={op[4] and op[4].count(0)}"
    if k in ("get", "get_small"):
        return f"{k} n={len(op[1])} addrs={op[1][:4]}... invalid={op[2] and op[2].count(0)}"
    if k in ("unset", "demote", "promote"):
        return f"{k} n={len(op[1])} addrs={op[1][:6]}..."
    if k == "invalidate":
        return f"invalidate u={op[1]} l=[{op[2]}, {op[3]}]"
    if k == "sample":
        return f"sample n={len(op[1])}"
    return k


# ---- census: the model alone ------------------------------------------------------------------------

@dataclass
class Census:
    events: dict = field(default_factory=dict)

    def hit(self, name: str):
        self.events[name] = self.events.get(name, 0) + 1


def census(cfg: MachineConfig, seed: int, oracle) -> dict:
    """Runs the log of `seed` through the model with the stand-in drop rule -> {event: times reached}.
    Only events the model can prove count: an overflow whose bytes certainly exceed the free arena,
    a rebuild whose tombstones certainly pass cap / 8, a demotion that certainly retires records."""
    m = Model(cfg, oracle)
    c = Census()
    compacted = demoted_after = False
    for op in gen_ops(cfg, seed):
        k = op[0]
        if k in ("put", "put_async"):
            pages = pages_of(cfg, op[2])
            drops = m.stand_in_drops(op[1], pages, op[4])
            if drops:
                c.hit("drop")
            m.put(op[1], pages, op[3], op[4], drops)
        elif k in ("get", "get_small"):
            m.get(op[1], op[2])
        elif k == "unset":
            m.unset(op[1])
        elif k == "invalidate":
            keyed_max = (m.cap + 2) // 64
            c.hit("inval_scan" if op[3] - op[2] >= keyed_max else "inval_keyed")
            m.invalidate(op[1], op[2], op[3])
            if m.rebuild_check():
                c.hit("rebuild")
        elif k == "compact":
            c.hit("compact")
            m.compact()
            compacted, demoted_after = True, False
            if m.rebuild_check():
                c.hit("rebuild")
        elif k == "demote":
            n, retired = m.demote(op[1])
            if retired:
                c.hit("wrap")
            if n and compacted:
                demoted_after = True
        elif k == "promote":
            if m.promote(op[1]) and demoted_after:
                c.hit("promote_after_demote_after_compact")
        elif k == "load":
            c.hit("load")
            m.load(cfg.load_slots, cfg.load_arena)
    return c.events
