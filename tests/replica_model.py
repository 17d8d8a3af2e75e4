"""The sequential model of one rank's replicated index (edge_fuse_b200/sharding.py, DESIGN.md §9).

Every rank stores its own chunks and imports the other ranks' exchange rows {u, l, position, owner,
stored length}.  Per store key (the FNV-1a-64 of the 16 address bytes) the model keeps:
  floor   the highest stream position the key has been claimed at: every valid put of this rank (also
          one the arena dropped) and every imported row that stored something;
  winner  (position, address, owner rank, page) of the record the key answers with, or None.
A put that stored its record, or an imported row, becomes the winner when its position is the key's
floor once every claim of its batch is in.  So the winner is the highest position among the rank's own
stored puts and the imported rows; a put or a row below the floor changes nothing.

Answers for an address a of key k (winner w):
  w is None                     MISS
  w.address == a                HIT (w.owner is this rank) or REMOTE(w.owner)
  w.address != a, w local       BAD_ENTRY (the reference's answer: the key holds another address)
  w.address != a, w remote      MISS      (a decision: DESIGN.md §9)
entries = keys with a local winner, remote_entries = keys with a remote winner.

unset(a) removes the key's winner when it is local, whatever address it holds, and leaves a remote
winner in place (a decision: DESIGN.md §9).  A key that was removed starts again from floor 0: the
table's tombstone keeps the old position but not the key, so the model only holds while every position
applied after an unset, a compaction or a table rebuild is above every position applied before it,
except a put below the floor of a key that still has a winner.
"""
from __future__ import annotations

MISS, HIT, BAD_ENTRY, REMOTE = 0, 1, 3, 5


def fnv_key(u: int, l: int) -> int:
    """FNV-1a-64 over the 16 little-endian bytes of {u, l}: the store key."""
    h = 14695981039346656037
    for b in int(u).to_bytes(8, "little") + int(l).to_bytes(8, "little"):
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


class Winner:
    __slots__ = ("pos", "addr", "owner", "page")

    def __init__(self, pos, addr, owner, page):
        self.pos, self.addr, self.owner, self.page = pos, addr, owner, page

    def __repr__(self):
        return f"Winner(pos={self.pos}, addr={self.addr}, owner={self.owner})"


class ReplicaModel:
    def __init__(self, rank: int):
        self.rank = rank
        self.floor = {}                  # key -> highest position claimed
        self.winner = {}                 # key -> Winner

    def _claim(self, key, pos):
        if pos > self.floor.get(key, -1):
            self.floor[key] = pos

    def put(self, chunks):
        """One put batch of this rank: chunks = [(addr, position, stored, page)]; addr None = an invalid
        address (claims nothing); stored = False for a put the arena dropped or a duplicate superseded
        inside the batch."""
        chunks = [c for c in chunks if c[0] is not None]
        for addr, pos, _, _ in chunks:
            self._claim(fnv_key(*addr), pos)
        for addr, pos, stored, page in chunks:
            key = fnv_key(*addr)
            if stored and self.floor[key] == pos:
                self.winner[key] = Winner(pos, addr, self.rank, page)

    def import_rows(self, rows):
        """One import of all-gathered rows [(addr, position, owner, stored)]: this rank's own rows and
        rows that stored nothing are skipped."""
        rows = [r for r in rows if r[2] != self.rank and r[3]]
        for addr, pos, _, _ in rows:
            self._claim(fnv_key(*addr), pos)
        for addr, pos, owner, _ in rows:
            key = fnv_key(*addr)
            if self.floor[key] == pos:
                self.winner[key] = Winner(pos, addr, owner, None)

    def unset(self, addrs):
        for addr in addrs:
            key = fnv_key(*addr)
            w = self.winner.get(key)
            if w is not None and w.owner == self.rank:
                del self.winner[key]
                self.floor.pop(key, None)

    def lookup(self, addr):
        """-> (status, owner rank or -1, page or None)."""
        w = self.winner.get(fnv_key(*addr))
        if w is None:
            return MISS, -1, None
        if w.addr != tuple(addr):
            return (BAD_ENTRY if w.owner == self.rank else MISS), -1, None
        if w.owner == self.rank:
            return HIT, -1, w.page
        return REMOTE, w.owner, None

    def entries(self) -> int:
        return sum(1 for w in self.winner.values() if w.owner == self.rank)

    def remote_entries(self) -> int:
        return sum(1 for w in self.winner.values() if w.owner != self.rank)

    def local_records(self) -> dict:
        """address -> page of every local winner: what a save of this rank holds."""
        return {w.addr: w.page for w in self.winner.values() if w.owner == self.rank}

    def remote_keys(self) -> list:
        return [w.addr for w in self.winner.values() if w.owner != self.rank]

    @classmethod
    def loaded(cls, rank: int, records: dict, pos: int = 0):
        """A fresh rank that loaded a file holding `records` (address -> page)."""
        m = cls(rank)
        m.put([(a, pos, True, p) for a, p in records.items()])
        return m
