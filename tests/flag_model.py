"""Every engine flag at once, restated over one store, for tests/test_gpu_flag_matrix.py and its CPU twin.

`FlagModel` composes the models that already exist, one per flag, and adds what they share:
  - a store, key -> (address, Record), keyed as the engine keys it (FNV-1a-64 of the 16 address bytes), so a
    request whose key holds another address is BAD_ENTRY, and unsets, evictions, demotions and promotions go
    by key (include/cachemap_b200.h);
  - each Record's decoded page, decided once by the oracle (oracle.lz4_decode; a consumed length other than
    compressed_length is BAD_DECODE) and, with VERIFY, whether oracle.fingerprint128 of that page equals the
    stored fingerprint (CORRUPT when not, unverified when there is none);
  - FREQ: admit_model.Sketch counts every valid request, whatever its answer;
  - GHOST: ghost_model.GhostTable, probed by exact misses only, filled by evictions, emptied by unsets,
    invalidations and renames of what they name;
  - VERIFY: verified / unverified / corrupt, counted for HIT and CORRUPT;
  - TOUCH: the records a call answers HIT (every record here is local, in the arena or the host tier);
  - host tier: hits counted for HIT only, and the addresses of those hits (the hot log, as a set).

`script(case, seed)` is one case's deterministic sequence: snapshot files written with oracle/snapshot.py
(damaged fingerprints, malformed blocks, raw records, a file without fingerprints), then about 60 steps of
puts, gets on every path, evictions, unsets, invalidations, renames, patches, demotions, promotions,
compaction and the calls that must count nothing.  The script does not depend on the flags, so one script
replays on an engine without them.

`CASES` is the matrix, and `kernels(case)` the get kernels a case launches, by the rule launch_get_small and
launch_decode (edge_fuse_b200/csrc/kernels.cu) choose them with.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import ef_oracle as O  # noqa: E402
from admit_model import Sketch, fnv_addr  # noqa: E402
from ghost_model import GhostTable  # noqa: E402
import key_edges  # noqa: E402

FINGERPRINT, VERIFY, TOUCH, FREQ, GHOST = 1, 2, 4, 8, 16           # CMB200_* (include/cachemap_b200.h)
MISS, HIT, INVALID, BAD_ENTRY, BAD_DECODE, CORRUPT = 0, 1, 2, 3, 4, 6
STATUS_NAMES = {MISS: "MISS", HIT: "HIT", INVALID: "INVALID", BAD_ENTRY: "BAD_ENTRY", BAD_DECODE: "BAD_DECODE",
                CORRUPT: "CORRUPT"}
PATHS = ("small", "tickets", "batch", "dev")
CAPACITY = 32                  # sketch width 32, halving period 320; ghost table of 256 entries

# ---- the matrix ---------------------------------------------------------------------------------

FLAG_LETTERS = ((VERIFY, "V"), (TOUCH, "T"), (FREQ, "F"), (GHOST, "G"))


def case_id(pshift: int, flags: int, ckpt0: bool = False) -> str:
    name = "".join(c for f, c in FLAG_LETTERS if flags & f) or "none"
    if flags & FINGERPRINT and not flags & VERIFY:
        name = "FP+" + name
    return f"p{pshift}-{name}" + ("-ckpt0" if ckpt0 else "")


def _cases():
    out = []
    for pshift in (16, 17):
        for bits in range(16):
            flags = sum(f for k, (f, _c) in enumerate(FLAG_LETTERS) if bits >> k & 1)
            out.append((pshift, flags, False))
        out.append((pshift, FINGERPRINT | TOUCH | FREQ | GHOST, False))
    out += [(12, 0, False), (12, VERIFY | TOUCH | FREQ | GHOST, False)]
    out += [(16, VERIFY | TOUCH | FREQ | GHOST, True), (17, VERIFY | TOUCH | FREQ | GHOST, True)]
    return [dict(id=case_id(*c), pshift=c[0], flags=c[1], ckpt0=c[2]) for c in out]


CASES = _cases()
GS_MAX_PAGE = 1 << 16          # k_get_small up to 64 KiB pages, k_get_small_pair above (kernels.cu)


def kernels(case) -> set:
    """The get kernels a case's script launches: launch_get_small picks the VERIFY variant when the engine
    keeps fingerprint tags (CMB200_VERIFY), TOUCH when it stamps, FREQ when it has a sketch; launch_decode
    picks k_decode_verify / _touch / _verify_touch the same way, for the batch gets."""
    f = case["flags"]
    v, t, q = bool(f & VERIFY), bool(f & TOUCH), bool(f & FREQ)
    name = "k_get_small" if (1 << case["pshift"]) <= GS_MAX_PAGE else "k_get_small_pair"
    dec = "k_decode" + ("_verify" if v else "") + ("_touch" if t else "")
    return {f"{name}<{str(v).lower()},{str(t).lower()},{str(q).lower()}>", dec}


# ---- records ------------------------------------------------------------------------------------

class Record:
    """A stored record: its address, its decoded page (None: the block does not decode to the page), whether
    a fingerprint is stored and whether it matches that page, its tier and its ts."""

    __slots__ = ("addr", "page", "has_fp", "fp_ok", "host", "ts")

    def __init__(self, addr, page, has_fp, fp_ok, ts):
        self.addr, self.page, self.has_fp, self.fp_ok, self.host, self.ts = tuple(addr), page, has_fp, fp_ok, False, ts


def decide_record(rec_bytes: bytes, bsize: int, fp):
    """(decoded page or None, fingerprint stored, fingerprint matches) of a record as a file holds it:
    24-byte prefix (compressed_length at bytes 16..19; 0 = raw page) + payload."""
    clen = int.from_bytes(rec_bytes[16:20], "little")
    payload = rec_bytes[24:]
    if clen == 0:
        page = bytes(payload[:bsize])
    else:
        page, used = O.lz4_decode(payload, bsize)
        if used != clen:
            return None, fp is not None, False
    return page, fp is not None, fp is not None and O.fingerprint128(page) == tuple(fp)


def page_of(a, version: int, bsize: int) -> np.ndarray:
    """A compressible page that names its address and version in its first 24 bytes."""
    rng = np.random.default_rng((a[0] * 1000003 + a[1]) * 131 + version)
    p = np.repeat(rng.integers(0, 256, size=bsize // 64, dtype=np.uint8), 64)
    p[:24] = np.frombuffer(np.array([a[0] & (2**64 - 1), a[1], version], dtype=np.uint64).tobytes(), dtype=np.uint8)
    return p


class FlagModel:
    def __init__(self, flags: int, pshift: int, capacity: int = CAPACITY):
        self.flags, self.bsize = flags, 1 << pshift
        self.verify = bool(flags & VERIFY)
        self.sketch = Sketch(capacity) if flags & FREQ else None
        self.ghosts = GhostTable(capacity) if flags & GHOST else None
        self.vstat = dict(verified=0, unverified=0, corrupt=0)
        self.tier_hits = 0
        self.hot: set = set()                  # tier hits since the last drain of the hot log
        self.store: dict = {}                  # key -> Record

    # -- lookups --
    def _rec(self, a):
        return self.store.get(fnv_addr(*a))

    def status(self, a):
        """(status, page or None, record or None) of one valid request."""
        r = self._rec(a)
        if r is None:
            return MISS, None, None
        if r.addr != tuple(a):
            return BAD_ENTRY, None, r
        if r.page is None:
            return BAD_DECODE, None, r
        if self.verify and r.has_fp and not r.fp_ok:
            return CORRUPT, None, r
        return HIT, r.page, r

    def entries(self) -> int:
        return len(self.store)

    # -- calls --
    def load(self, records, with_fp: bool):
        for ts, hi, lo, rec in records:
            a = (int.from_bytes(rec[0:8], "little"), int.from_bytes(rec[8:16], "little"))
            page, has_fp, ok = decide_record(rec, self.bsize, (hi, lo) if with_fp else None)
            self.store[fnv_addr(*a)] = Record(a, page, has_fp, ok, ts)

    def put(self, addrs, pages, ts):
        for a, p, t in zip(addrs, pages, ts):
            self.store[fnv_addr(*a)] = Record(a, bytes(p.tobytes()), True, True, int(t))

    def get(self, addrs, valid=None):
        """One counting launch.  -> (statuses, {index: page} of the hits, keys answered HIT)."""
        st, pages, hit_keys, probe, counted = [], {}, set(), [], []
        for i, a in enumerate(addrs):
            if valid is not None and not valid[i]:
                st.append(INVALID)
                continue
            counted.append(fnv_addr(*a))
            s, page, r = self.status(a)
            st.append(s)
            if s == HIT:
                pages[i] = page
                hit_keys.add(fnv_addr(*a))
                if r.host:
                    self.tier_hits += 1
                    self.hot.add(tuple(a))
            if self.verify and s in (HIT, CORRUPT):
                self.vstat["corrupt" if s == CORRUPT else "verified" if r.has_fp else "unverified"] += 1
            if s == MISS:
                probe.append(tuple(a))
        if self.sketch is not None:
            self.sketch.launch(counted)
        if self.ghosts is not None:
            self.ghosts.probe(probe)
        return st, pages, hit_keys

    def evict(self, addrs) -> int:
        """cmb200_evict_batch (or, without GHOST, cmb200_unset_batch): by key; a ghost for each address whose
        own record the call removed, the first of repeats, in array order."""
        own = []
        for a in addrs:
            r = self._rec(a)
            if r is not None and r.addr == tuple(a) and tuple(a) not in own:
                own.append(tuple(a))
        for a in addrs:
            self.store.pop(fnv_addr(*a), None)
        if self.ghosts is not None:
            self.ghosts.insert(own)
        return len(own)

    def unset(self, addrs):
        for a in addrs:
            self.store.pop(fnv_addr(*a), None)
        if self.ghosts is not None:
            self.ghosts.remove(addrs)

    def _span(self, u, lo, hi):
        return [k for k, r in self.store.items() if r.addr[0] == u and lo <= r.addr[1] <= hi]

    def invalidate(self, u, lo, hi) -> int:
        ks = self._span(u, lo, hi)
        for k in ks:
            del self.store[k]
        if self.ghosts is not None:
            self.ghosts.remove_span(u, lo, hi)
        return len(ks)

    def rename(self, uf, ut, lo, hi) -> int:
        ks = self._span(uf, lo, hi)
        moved = [self.store.pop(k) for k in ks]
        for r in moved:
            r.addr = (ut, r.addr[1])
            r.host = False                     # records of the host tier move into the arena
            self.store[fnv_addr(*r.addr)] = r
        if self.ghosts is not None:
            self.ghosts.remove_span(uf, lo, hi)
            self.ghosts.remove_span(ut, lo, hi)
        return len(moved)

    def patch(self, addrs, offs, datas, ts):
        """Distinct addresses.  A patch is a put: no get counter moves."""
        out = []
        for a, o, d, t in zip(addrs, offs, datas, ts):
            s, page, r = self.status(a)
            if s == HIT:
                p = bytearray(page)
                p[o:o + len(d)] = d
                self.store[fnv_addr(*a)] = Record(a, bytes(p), True, True, int(t))
            elif s in (BAD_DECODE, CORRUPT):
                del self.store[fnv_addr(*a)]
            out.append(s)
        return out

    def demote(self, addrs) -> int:
        n = 0
        for a in addrs:
            r = self._rec(a)
            if r is not None and not r.host:
                r.host = True
                n += 1
        return n

    def promote(self, addrs) -> int:
        n = 0
        for a in addrs:
            r = self._rec(a)
            if r is not None and r.host:
                r.host = False
                n += 1
        return n

    def drain_hot(self) -> set:
        h, self.hot = self.hot, set()
        return h


# ---- one case's script --------------------------------------------------------------------------

SPECIAL_U, MALFORMED_U, NEVER_U = 21, 22, 14
POOL_U = (11, 12, 13)
POOL_L = 16
GET_LANES = 32                 # cmb200_engine::GET_LANES: small gets in flight at once (engine.cu)
LANE_REPS = 16


def _edges():
    g = key_edges.load()["groups"]
    return [g["pair0"][0], g["pair0"][1], g["key0"][0], g["key0"][1], g["key_ones"][0], g["key_ones"][1]]


def _first_offset_at(block: bytes) -> int:
    tok = block[0]
    ip, lit = 1, tok >> 4
    if lit == 15:
        while True:
            b = block[ip]
            ip += 1
            lit += b
            if b != 255:
                break
    return ip + lit


def _files(pshift: int, seed: int):
    """Two snapshot files' records, (ts, fp_hi, fp_lo, record bytes):
    A, with fingerprints: compressed records (0..5 clean, 6..9 with a damaged fingerprint) and raw records
       (compressed_length 0: 10, 11 clean, 12 damaged), all at u = SPECIAL_U;
    B, without fingerprints: 8 malformed blocks with valid lengths (0..7, altered as the malformed-block
       test of tests/test_gpu_get_small_128k.py alters them) and 4 clean blocks (8..11), at u = MALFORMED_U."""
    bs = 1 << pshift
    rng = np.random.default_rng(seed)
    a_recs, b_recs = [], []
    for i in range(13):
        a = (SPECIAL_U, i)
        page = page_of(a, 0, bs)
        if i < 10:
            blk = O.lz4_encode(page)
            rec = O.record_prefix(*a, len(blk)) + blk
        else:
            rec = O.record_prefix(*a, 0) + page.tobytes()
        hi, lo = O.fingerprint128(page)
        if i in (6, 7, 8, 9, 12):
            lo ^= 1 << (i % 64)
        a_recs.append((1000 + i, hi, lo, rec))
    for i in range(12):
        a = (MALFORMED_U, i)
        blk = bytearray(O.lz4_encode(page_of(a, 0, bs)))
        if i < 8:
            kind = i % 4
            if kind == 0:                                 # an offset that points before the page
                at = _first_offset_at(bytes(blk))
                if at + 2 <= len(blk):
                    blk[at:at + 2] = (0xffff).to_bytes(2, "little")
            elif kind == 1:                               # length bytes: token nibbles and extension bytes
                blk[0] = 0xff
                blk[1] = int(rng.integers(0, 256))
            elif kind == 2:                               # truncated last literals
                blk = blk[:-3]
            else:                                         # a few random bytes
                for p in rng.integers(0, len(blk), 4):
                    blk[int(p)] = int(rng.integers(0, 256))
        b_recs.append((2000 + i, 0, 0, O.record_prefix(*a, len(blk)) + bytes(blk)))
    return [(a_recs, True), (b_recs, False)]


def script(case, seed: int = 0, steps: int = 60, lane_reps: int = LANE_REPS):
    """-> (files, ops).  files: [(records, with_fingerprints)], loaded first in order.  ops: tuples, the
    first item naming the call:
      ("put", addrs, version, ts)            ("get", path, [addrs, ...], valid or None)  path in PATHS;
      ("evict", addrs)  ("unset", addrs)      "tickets" has several lists, begun in order, ended in `order`
      ("inv", u, lo, hi)  ("rename", uf, ut, lo, hi)  ("patch", addrs, offs, datas, ts)
      ("demote", addrs)  ("promote", addrs)  ("compact",)  ("sample",)  ("locate", addrs)  ("read", addrs)
      ("get", "lanes", [addrs, ...], held): the first `held` lists are begun and left outstanding, every later
      one is begun and ended in turn, then the held ones are ended
    Nothing in it depends on the flags."""
    pshift = case["pshift"]
    bs = 1 << pshift
    rng = random.Random(pshift * 1000 + seed)
    files = _files(pshift, seed + pshift)
    special = [(SPECIAL_U, i) for i in range(13)] + [(MALFORMED_U, i) for i in range(12)]
    pool = [(u, l) for u in POOL_U for l in range(POOL_L)]
    never = [(NEVER_U, l) for l in range(8)]
    edges = _edges()
    ops = []
    gone: list = []
    live: set = set()                      # pool addresses the script has put (for its own choices only)
    version = [0]
    tsv = [10]
    path_turn = [0]
    asked = [False]                        # pair0[0] asked for after pair0[1] took its key

    def put(addrs):
        version[0] += 1
        ts = []
        for a in addrs:
            tsv[0] += 1
            ts.append(tsv[0])
            live.add(a)
        ops.append(("put", list(addrs), version[0], ts))

    def get():
        path = PATHS[path_turn[0] % len(PATHS)]
        path_turn[0] += 1
        addrs = (rng.sample(special, 9) + rng.sample(pool, 7) + rng.sample(never, 2)
                 + rng.sample(edges if asked[0] else edges[1:], 2) + (rng.sample(gone, min(3, len(gone))) if gone else []))
        addrs.insert(4, addrs[0])          # repeats within one call
        addrs.insert(11, addrs[12])
        rng.shuffle(addrs)
        if path == "tickets":
            cut = sorted(rng.sample(range(1, len(addrs)), 2))
            parts = [addrs[:cut[0]], addrs[cut[0]:cut[1]], addrs[cut[1]:]]
            order = rng.choice([(2, 0, 1), (1, 2, 0), (2, 1, 0)])
            ops.append(("get", path, parts, order))
            return
        valid = None
        if path != "small" and rng.random() < 0.5:           # the fused get takes no mask
            valid = [1] * len(addrs)
            for k in rng.sample(range(len(addrs)), 2):
                valid[k] = 0
        ops.append(("get", path, [addrs], valid))

    put(pool[:36] + [edges[0], edges[2], edges[4]])
    ops.append(("demote", special[::2]))
    fixed = {3: ("evict", [edges[0]]), 5: "put_edge", 7: "get_edge"}
    for step in range(steps):
        if step in fixed:
            f = fixed[step]
            if f == "put_edge":
                put([edges[1]])            # pair0[1] takes the key pair0[0] left a ghost of
            elif f == "get_edge":
                ops.append(("get", "batch", [[edges[0], edges[1], edges[0]] + rng.sample(pool, 4)], None))
                ops.append(("get", "small", [[edges[0], edges[3], edges[5]] + rng.sample(special, 4)], None))
                # until here no get asks for pair0[0] and no unset names it, so its ghost is there to survive
                asked[0] = True
                gone.append(edges[0])
            else:
                ops.append(f)
            continue
        op = rng.choice(["get"] * 8 + ["put", "evict", "evict", "unset", "inv", "inv_scan", "rename", "patch",
                         "demote", "demote", "promote", "promote", "compact", "quiet"])
        if op == "get":
            get()
        elif op == "put":
            put(rng.sample(pool, 10))
        elif op == "evict":
            addrs = rng.sample(pool, 6) + rng.sample(never, 1)
            addrs.insert(2, addrs[0])
            ops.append(("evict", addrs))
            gone.extend(a for a in addrs if a in live)
            live.difference_update(addrs)
        elif op == "unset":
            addrs = rng.sample(pool, 3) + rng.sample(gone, min(2, len(gone)))
            ops.append(("unset", addrs))
            live.difference_update(addrs)
        elif op in ("inv", "inv_scan"):
            u = rng.choice(POOL_U)
            lo = rng.randrange(POOL_L - 4)
            hi = lo + (rng.randrange(3) if op == "inv" else 200)      # by key, or by a scan of the table
            ops.append(("inv", u, lo, hi))
        elif op == "rename":
            uf, ut = rng.sample(POOL_U, 2)
            lo = rng.randrange(POOL_L - 4)
            ops.append(("rename", uf, ut, lo, lo + rng.randrange(4)))
        elif op == "patch":
            addrs = rng.sample(pool, 4) + rng.sample(never, 1)
            offs = [rng.randrange(bs - 8) for _ in addrs]
            tsv[0] += 1
            ops.append(("patch", addrs, offs, [bytes([0x5A, len(ops) & 0xFF, 3]) for _ in addrs], [tsv[0]] * len(addrs)))
        elif op == "demote":
            ops.append(("demote", rng.sample(special, 8) + rng.sample(pool, 4)))
        elif op == "promote":
            ops.append(("promote", rng.sample(special, 8) + rng.sample(pool, 4)))
        elif op == "compact":
            ops.append(("compact",))
        else:
            ops.append(rng.choice([("sample",), ("locate", rng.sample(special + pool, 12)),
                                   ("read", rng.sample(special + pool, 6))]))
    # ghosts that an unset, an invalidation and a rename remove
    four = [(POOL_U[2], l) for l in range(4)]
    put(four)
    ops += [("evict", four), ("unset", four[:1]), ("inv", POOL_U[2], 1, 1), ("rename", POOL_U[2], POOL_U[0], 2, 2)]
    gone += four
    # every path asks for every loaded record with each half of them in the host tier, so that every answer
    # comes from both tiers on every path whatever the random steps left where; then evicted pages again
    for half in (special[::2], special[1::2]):
        ops.append(("demote", half))
        ops.append(("promote", [a for a in special if a not in half]))
        for path in PATHS:
            addrs = special + rng.sample(never, 2) + rng.sample(gone, min(4, len(gone)))
            ops.append(("get", path, [addrs[:9], addrs[9:20], addrs[20:]] if path == "tickets" else [addrs],
                        (1, 2, 0) if path == "tickets" else None))
    # small gets that wait for a lane's previous probe: every lane but one held by an outstanding ticket, so
    # that the gets after them all run on the one free lane, each begun as soon as the one before has ended
    held = [[a] for a in rng.sample(special, 12) + rng.sample(pool, 12) + rng.sample(never, 4) + rng.sample(gone, 3)]
    again = [rng.sample(special, 4) + rng.sample(gone, 2) + rng.sample(never, 1) for _ in range(lane_reps)]
    assert len(held) == GET_LANES - 1
    ops.append(("get", "lanes", held + again, len(held)))
    # last: patches of every loaded record, so that the patch path meets malformed and corrupt records in
    # both tiers, then one get of all of them (what is left)
    tsv[0] += 1
    ops.append(("patch", special, [8] * len(special), [b"\xa5\x5a"] * len(special), [tsv[0]] * len(special)))
    ops.append(("get", "batch", [special + pool[:8]], None))
    return files, ops


def run(case, seed: int = 0, steps: int = 60, flags=None, census=None):
    """The model alone over a case's script.  census (a set) collects (path, status, tier) of every answer:
    tier "arena", "host" or "-" for answers without a record of the address.  -> the model."""
    files, ops = script(case, seed, steps)
    m = FlagModel(case["flags"] if flags is None else flags, case["pshift"])
    for recs, with_fp in files:
        m.load(recs, with_fp)
    for op in ops:
        apply(m, op, census)
    return m


def apply(m: FlagModel, op, census=None):
    """Applies one op to the model -> what the call returns (statuses, counts), for the tests to compare."""
    kind = op[0]
    if kind == "put":
        _, addrs, version, ts = op
        m.put(addrs, [page_of(a, version, m.bsize) for a in addrs], ts)
        return None
    if kind == "get":
        _, path, parts, extra = op
        out = []
        for part in parts:
            valid = extra if path in ("batch", "dev") else None
            if census is not None:
                for i, a in enumerate(part):
                    if valid is not None and not valid[i]:
                        census.add((path, INVALID, "-"))
                        continue
                    s, _p, r = m.status(a)
                    census.add((path, s, "host" if r is not None and r.host and s != BAD_ENTRY else
                                "arena" if r is not None and s != BAD_ENTRY else "-"))
            out.append(m.get(part, valid))
        return out
    if kind == "evict":
        return m.evict(op[1]) if m.ghosts is not None else m.unset(op[1])
    if kind == "unset":
        return m.unset(op[1])
    if kind == "inv":
        return m.invalidate(*op[1:])
    if kind == "rename":
        return m.rename(*op[1:])
    if kind == "patch":
        return m.patch(*op[1:])
    if kind == "demote":
        return m.demote(op[1])
    if kind == "promote":
        return m.promote(op[1])
    return None                                  # compact, sample, locate, read: nothing moves
