"""The snapshot-chain format of tests/snapshot_chain.py without a GPU: round trips of bases and deltas,
and replay_chain against a dict model of the store over seeded random operation sequences — puts,
rewrites, unsets, addresses that share a store key and addresses whose key is a sentinel (0, ~0) —
written tick by tick the way the engine writes them: tombstones for the addresses live at the previous
tick and not now, records for the keys put since the previous tick's watermark."""
import os
import random
import struct

import pytest

import key_edges
import snapshot_chain as sc
from oracle import ef_oracle, snapshot

PSHIFT = 12


def _rec(u, l, payload: bytes):
    """A record in the base's format: 24-byte prefix {u, l, compressed_length, 0} + payload (raw here)."""
    return struct.pack("<QQiI", u, l, 0, 0) + payload


def test_base_round_trip_keeps_a_zero_chain_id_byte_identical(tmp_path):
    recs = [(7, 1, 2, _rec(1, 2, b"a" * 40)), (9, 0, 0, _rec(3, 4, b"b" * 33))]
    plain, chained = str(tmp_path / "plain"), str(tmp_path / "chained")
    snapshot.write_snapshot(plain, PSHIFT, recs, True)
    sc.write_base(chained, PSHIFT, recs, 0, True)
    assert open(plain, "rb").read() == open(chained, "rb").read()
    assert sc.read_chain_id(chained) == 0
    sc.write_base(chained, PSHIFT, recs, 0xDEADBEEF12345678, True)
    assert sc.read_chain_id(chained) == 0xDEADBEEF12345678
    assert snapshot.read_snapshot(chained) == (PSHIFT, 1, recs)


def test_delta_round_trip_and_truncation(tmp_path):
    recs = [(5, 6, 7, _rec(10, 11, bytes(range(200)))), (8, 0, 0, _rec(12, 13, b"z" * 17))]
    p = str(tmp_path / "base.d1")
    sc.write_delta(p, PSHIFT, 42, 1, [(1, 2), (3, 4)], recs, True)
    d = sc.read_delta(p)
    assert (d["pshift"], d["chain"], d["index"], d["flags"]) == (PSHIFT, 42, 1, 1)
    assert d["tombstones"] == [(1, 2), (3, 4)] and d["records"] == recs
    raw = open(p, "rb").read()
    assert len(raw) == 64 + 32 + sum(32 + (len(r[3]) + 15) // 16 * 16 for r in recs)
    for cut in (10, 64 + 8, len(raw) - 1):
        open(p, "wb").write(raw[:cut])
        with pytest.raises(ValueError):
            sc.read_delta(p)
    open(p, "wb").write(raw + b"\0" * 16)
    with pytest.raises(ValueError):
        sc.read_delta(p)


class _Sim:
    """A store of one record per key (the last put wins), with the engine's stream sequence: a put
    raises its key's seq, so 'put since the last tick' is seq >= that tick's watermark."""

    def __init__(self):
        self.rec = {}            # key -> (addr, record tuple, seq)
        self.seq = 1
        self.w = None            # watermark and live addresses of the last tick
        self.base_live = set()
        self.k = 0

    def put(self, addr, payload: bytes):
        key = sc_key(addr)
        self.rec[key] = (addr, (self.seq, 0, 0, _rec(addr[0], addr[1], payload)), self.seq)
        self.seq += 1

    def unset(self, addr):
        self.rec.pop(sc_key(addr), None)

    def state(self):
        return {a: r for a, r, _s in self.rec.values()}

    def tick(self, base_path, chain_id):
        live = set(self.state())
        if self.w is None:
            sc.write_base(base_path, PSHIFT, [r for _a, r, _s in self.rec.values()], chain_id)
        else:
            self.k += 1
            tombs = sorted(self.base_live - live)
            recs = [r for _a, r, s in self.rec.values() if s >= self.w]
            sc.write_delta(f"{base_path}.d{self.k}", PSHIFT, chain_id, self.k, tombs, recs)
        self.w, self.base_live = self.seq, live


def sc_key(addr):
    return ef_oracle.addr_key(*addr)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_replay_chain_matches_the_store_at_every_tick(tmp_path, seed, oracle):
    rnd = random.Random(seed)
    fx = key_edges.load()
    pool = list(fx["ordinary"][:24])
    for g in fx["groups"].values():
        pool += list(g)
    sim = _Sim()
    base = str(tmp_path / "c.snap")
    for a in pool[::2]:
        sim.put(a, bytes([rnd.randrange(256)]) * rnd.randrange(1, 90))
    sim.tick(base, 77)
    history = [sim.state()]
    for _ in range(8):
        for _ in range(rnd.randrange(0, 30)):
            a = rnd.choice(pool)
            if rnd.random() < 0.25:
                sim.unset(a)
            else:
                sim.put(a, bytes([rnd.randrange(256)]) * rnd.randrange(1, 90))
        sim.tick(base, 77)
        history.append(sim.state())
        state, k = sc.replay_chain(base)
        assert k == sim.k and state == history[-1]
    # a delta with nothing changed is empty
    sim.tick(base, 77)
    d = sc.read_delta(f"{base}.d{sim.k}")
    assert d["tombstones"] == [] and d["records"] == []
    history.append(sim.state())
    # crash shapes: the valid run ends at the first bad delta, and the store is the one of that tick
    os.rename(f"{base}.d3", f"{base}.gone")
    assert sc.replay_chain(base) == (history[2], 2)
    os.rename(f"{base}.gone", f"{base}.d3")
    raw = open(f"{base}.d5", "rb").read()
    open(f"{base}.d5", "wb").write(raw[:-1])
    assert sc.replay_chain(base) == (history[4], 4)
    open(f"{base}.d5", "wb").write(raw)
    d = sc.read_delta(f"{base}.d2")
    sc.write_delta(f"{base}.d2", PSHIFT, 78, 2, d["tombstones"], d["records"])
    assert sc.replay_chain(base) == (history[1], 1)
    sc.write_delta(f"{base}.d2", PSHIFT, 77, 3, d["tombstones"], d["records"])
    assert sc.replay_chain(base) == (history[1], 1)
