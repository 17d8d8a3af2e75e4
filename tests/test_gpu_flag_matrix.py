"""GPU tests of the engine's flags together: every subset of VERIFY, TOUCH, FREQ and GHOST against one
composed model (tests/flag_model.py), compared exactly after every step.

Each case of flag_model.CASES runs its seeded script on an engine with a host tier: snapshot files with
damaged fingerprints, malformed blocks, raw records and no fingerprints; puts; gets on every path (the fused
get, several begin / end tickets ended out of order, the batch get to the host and to the device with `valid`
masks); evictions, unsets, invalidations, renames, patches, demotions, promotions, compaction, and sampling,
lookups and record reads, which count nothing.  After every step: every status, the bytes of every hit, a
canary in the fused get's output of every other answer, the verified-read counters, the sketch, the ghost
table, tier hits and the hot log, entries and, with TOUCH, every record's ts.  The same script on an engine
without flags answers the same, CORRUPT aside.  Then every fused-get variant at full occupancy."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import admit_model as A
import flag_model as M
from oracle import snapshot

pytestmark = pytest.mark.gpu

CANARY = 0xC3
TIER_BYTES = 64 << 20


def coarse_ns() -> int:
    """CLOCK_REALTIME_COARSE in ns, the clock CMB200_TOUCH stamps with."""
    ts = (C.c_long * 2)()
    assert C.CDLL(None).clock_gettime(5, ts) == 0
    return ts[0] * 1_000_000_000 + ts[1]


class Ticket(C.Structure):
    _fields_ = [("lane", C.c_int), ("n", C.c_uint32), ("status", C.POINTER(C.c_int32))]

    def __init__(self):
        super().__init__(-1, 0, None)                  # nothing in flight until a begin fills it


def _arrays(addrs):
    return (np.array([a[0] for a in addrs], dtype=np.uint64), np.array([a[1] for a in addrs], dtype=np.uint64))


def _addr(addrs):
    return np.ascontiguousarray(np.array([[a[0], a[1]] for a in addrs], dtype=np.uint64))


class _Pinned:
    """Page-locked output pages prefilled with the canary."""

    def __init__(self, E, n, bs):
        self.L, self.n, self.bs = E.lib(), n, bs
        self.p = self.L.cmb200_host_alloc(max(1, n) * bs)
        assert self.p
        C.memset(self.p, CANARY, n * bs)

    def pages(self):
        return np.ctypeslib.as_array((C.c_uint8 * (self.n * self.bs)).from_address(self.p)).reshape(self.n, self.bs).copy()

    def free(self):
        self.L.cmb200_host_free(self.p)


def _begin(E, e, addrs, buf):
    addr = _addr(addrs)                   # alive across the call: begin copies the addresses out of it
    t = Ticket()
    assert E.lib().cmb200_get_small_begin(e.h, len(addrs), addr.ctypes.data, buf.p, C.byref(t)) == 0, E.last_error()
    return t


def _end(E, e, t, n):
    st = np.zeros(n, dtype=np.int32)
    assert E.lib().cmb200_get_small_end(e.h, C.byref(t), st.ctypes.data) == 0, E.last_error()
    return st


def _get(E, e, path, parts, extra):
    """-> [(pages, statuses)] per part, and whether the outputs of the non-hits are canaries.
    tickets: every part begun, then ended in the order `extra`.  lanes: the first `extra` parts begun and left
    outstanding, each later part begun and ended in turn, then the held ones ended."""
    L, bs = E.lib(), e.bsize
    if path == "small":
        (addrs,) = parts
        buf = _Pinned(E, len(addrs), bs)
        try:
            addr = _addr(addrs)
            st = np.zeros(len(addrs), dtype=np.int32)
            assert L.cmb200_get_small(e.h, len(addrs), addr.ctypes.data, buf.p, st.ctypes.data) == 0, E.last_error()
            return [(buf.pages(), st)], True
        finally:
            buf.free()
    if path in ("tickets", "lanes"):
        bufs, tickets, out = [], [], [None] * len(parts)
        try:
            if path == "tickets":
                for addrs in parts:                               # begun in order, all outstanding at once
                    bufs.append(_Pinned(E, len(addrs), bs))
                    tickets.append(_begin(E, e, addrs, bufs[-1]))
                order = extra                                     # ended out of order
            else:
                for addrs in parts[:extra]:
                    bufs.append(_Pinned(E, len(addrs), bs))
                    tickets.append(_begin(E, e, addrs, bufs[-1]))
                bufs += [_Pinned(E, len(p), bs) for p in parts[extra:]]
                tickets += [Ticket() for _ in parts[extra:]]
                errors = []

                def turns(ks):
                    # two threads take turns on the one lane left: a begin that spins for the lane takes it as
                    # soon as the other's end frees it, often before that get's ghost probe has run
                    try:
                        for k in ks:
                            tickets[k] = _begin(E, e, parts[k], bufs[k])
                            st = _end(E, e, tickets[k], len(parts[k]))
                            out[k] = (bufs[k].pages(), st)
                    except Exception as x:                       # raised again below, on the test's thread
                        errors.append(x)
                ks = range(extra, len(parts))
                th = [threading.Thread(target=turns, args=(ks[j::2],)) for j in range(2)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                if errors:
                    raise errors[0]
                order = range(extra - 1, -1, -1)
            for k in order:
                st = _end(E, e, tickets[k], len(parts[k]))
                out[k] = (bufs[k].pages(), st)
            return out, True
        finally:
            for t in tickets:                                     # a failed check leaves no lane taken
                if t.lane >= 0:
                    L.cmb200_get_small_end(e.h, C.byref(t), None)
            for b in bufs:
                b.free()
    (addrs,) = parts
    u, l = _arrays(addrs)
    valid = None if extra is None else np.array(extra, dtype=np.uint8)
    if path == "batch":
        return [e.get(u, l, valid=valid)], False
    n = len(addrs)
    dev = e.dev_alloc(n * bs)
    try:
        out = np.zeros((n, bs), dtype=np.uint8)
        st = np.zeros(n, dtype=np.int32)
        addr = _addr(addrs)
        v = None if valid is None else np.ascontiguousarray(valid)
        assert L.cmb200_get_batch_dev(e.h, n, addr.ctypes.data, None if v is None else v.ctypes.data, dev,
                                      st.ctypes.data) == 0, E.last_error()
        e.d2h(out, dev)
        return [(out, st)], False
    finally:
        e.dev_free(dev)


def _ts_all(e, path):
    e.save(path)
    return {(int.from_bytes(r[0:8], "little"), int.from_bytes(r[8:16], "little")): ts
            for ts, _h, _l, r in snapshot.read_snapshot(path)[2]}


def _check_state(E, e, m, flags, where):
    vs = e.verify_stats()
    want = m.vstat if flags & M.VERIFY else dict(verified=0, unverified=0, corrupt=0)
    assert {k: vs[k] for k in want} == want and vs["scanned"] == 0, (where, vs, want)
    if m.sketch is not None:
        sk = m.sketch
        assert (e.freq_read() == sk.words()).all(), where
        st = e.freq_stats()
        assert (st["width"], st["period"], st["increments"], st["since_halving"], st["halvings"]) == \
            (sk.width, sk.period, sk.increments, sk.since, sk.halvings), (where, st)
    if m.ghosts is not None:
        tab, want_tab = e.ghost_read(), m.ghosts.words()
        bad = np.nonzero((tab != want_tab).any(axis=1))[0]
        assert len(bad) == 0, (where, bad[:4], tab[bad[:4]], want_tab[bad[:4]])
        gs = e.ghost_stats()
        for k, v in m.ghosts.stats().items():
            assert gs[k] == v, (where, k, gs[k], v)
    ts = e.host_tier_stats()
    assert ts["hits"] == m.tier_hits and ts["retired_records"] == 0, (where, ts["hits"], m.tier_hits)
    hu, hl, lost = e.tier_hot()
    assert lost == 0 and {(int(a), int(b)) for a, b in zip(hu, hl)} == m.drain_hot(), where
    assert e.entries() == m.entries(), (where, e.entries(), m.entries())


def _run(E, case, flags, tmp_path, monkeypatch, seed=0, lane_reps=M.LANE_REPS):
    """One case's script on a fresh engine with `flags`, against the model of the same flags after every
    step.  -> [(statuses, {i: page}) of every get part] for the replay comparison."""
    pshift = case["pshift"]
    bs = 1 << pshift
    if case["ckpt0"]:
        monkeypatch.setenv("CMB200_CKPT", "0")                    # no parse checkpoints: the one-warp walk
    else:
        monkeypatch.delenv("CMB200_CKPT", raising=False)
    files, ops = M.script(case, seed, lane_reps=lane_reps)
    e = E.Engine(pshift=pshift, capacity=M.CAPACITY, arena_bytes=256 << 20, table_slots=1024, max_batch=64,
                 flags=flags, host_tier_bytes=TIER_BYTES)
    m = M.FlagModel(flags, pshift)
    touch = bool(flags & M.TOUCH)
    snap_ts = str(tmp_path / f"ts{flags}.snap")
    answers = []
    try:
        for k, (recs, with_fp) in enumerate(files):
            path = str(tmp_path / f"f{k}.snap")
            snapshot.write_snapshot(path, pshift, recs, with_fingerprints=with_fp)
            assert e.load(path) == len(recs)
            m.load(recs, with_fp)
        _check_state(E, e, m, flags, "load")
        for step, op in enumerate(ops):
            where = (case["id"], flags, step, op[0], op[1] if op[0] == "get" else None)
            kind = op[0]
            t0 = coarse_ns()
            if kind == "get":
                got, canaries = _get(E, e, op[1], op[2], op[3])
                t1 = coarse_ns()
                hit_keys = set()
                want = M.apply(m, op)
                for (pages, st), (wst, wpages, keys), part in zip(got, want, op[2]):
                    assert st.tolist() == wst, (where, part, st.tolist(), wst)
                    for i, s in enumerate(wst):
                        if s == M.HIT:
                            assert pages[i].tobytes() == wpages[i], (where, i, part[i])
                        elif canaries:
                            # the fused get writes a page only on HIT; CORRUPT pages are never written out
                            assert (pages[i] == CANARY).all(), (where, i, part[i], s)
                    answers.append((st.copy(), {i: pages[i].tobytes() for i in wpages}))
                    hit_keys |= keys
            else:
                hit_keys = set()
                if kind == "put":
                    _, addrs, version, tsv = op
                    e.put(*_arrays(addrs), np.stack([M.page_of(a, version, bs) for a in addrs]), ts=tsv)
                    M.apply(m, op)
                elif kind == "evict":
                    if flags & M.GHOST:
                        assert e.evict(*_arrays(op[1])) == M.apply(m, op), where
                    else:
                        e.unset(*_arrays(op[1]))
                        M.apply(m, op)
                elif kind == "unset":
                    e.unset(*_arrays(op[1]))
                    M.apply(m, op)
                elif kind == "inv":
                    assert e.invalidate(*op[1:]) == M.apply(m, op), where
                elif kind == "rename":
                    moved, dropped = e.rename(*op[1:])
                    assert dropped == 0 and moved == M.apply(m, op), where
                elif kind == "patch":
                    _, addrs, offs, datas, tsv = op
                    st = e.patch(*_arrays(addrs), offs, datas, ts=tsv)
                    assert st.tolist() == M.apply(m, op), (where, st.tolist())
                elif kind == "demote":
                    assert e.demote(*_arrays(op[1])) == M.apply(m, op), where
                elif kind == "promote":
                    assert e.promote(*_arrays(op[1])) == M.apply(m, op), where
                elif kind == "compact":
                    e.compact()
                elif kind == "sample":
                    e.sample([(k * 0x9E3779B97F4A7C15) % (1 << 63) for k in range(64)])
                elif kind == "locate":
                    st, _ = e.locate(*_arrays(op[1]))
                    want = [{M.MISS: M.MISS, M.BAD_ENTRY: M.BAD_ENTRY}.get(m.status(a)[0], M.HIT) for a in op[1]]
                    assert st.tolist() == want, where
                elif kind == "read":
                    lens = e.read_records_raw(*_arrays(op[1]))[1]
                    assert [int(x) >= 0 for x in lens] == [m.status(a)[0] not in (M.MISS, M.BAD_ENTRY)
                                                             for a in op[1]], where
                t1 = coarse_ns()
            _check_state(E, e, m, flags, where)
            if touch:
                got_ts = _ts_all(e, snap_ts)
                assert set(got_ts) == {r.addr for r in m.store.values()}, where
                for key, r in m.store.items():
                    ts = got_ts[r.addr]
                    if key in hit_keys:
                        assert ts >= r.ts and t0 <= ts <= t1, (where, r.addr, ts, r.ts, t0, t1)
                        r.ts = ts
                    else:
                        assert ts == r.ts, (where, r.addr, ts, r.ts)
        if not flags & M.FREQ:
            with pytest.raises(RuntimeError, match="CMB200_FREQ"):
                e.freq_stats()
        if not flags & M.GHOST:
            with pytest.raises(RuntimeError, match="CMB200_GHOST"):
                e.ghost_stats()
            return answers, None
        return answers, e.ghost_stats()["lane_waits"]
    finally:
        e.close()


@pytest.mark.parametrize("case", M.CASES, ids=[c["id"] for c in M.CASES])
def test_every_flag_combination_follows_the_model_after_every_step(E, gpu, oracle, tmp_path, monkeypatch, case):
    """Also pins the batch get's tier accounting: a host-tier record answered BAD_DECODE or CORRUPT by
    cmb200_get_batch(_dev) is a miss, so it is not a tier hit and is not logged as hot (decode_request used to
    book both before the decode decided)."""
    with_flags, waits = _run(E, case, case["flags"], tmp_path, monkeypatch)
    print(f"{case['id']}: lane waits {waits}")
    if case["flags"] == 0:
        return
    # Flags do not change answers: the same script without them, CORRUPT read as HIT.  The script's last get
    # follows patches that remove CORRUPT records only under VERIFY, so it is left out.
    without, _ = _run(E, case, 0, tmp_path, monkeypatch)
    assert len(with_flags) == len(without)
    for k, ((s1, p1), (s2, p2)) in enumerate(zip(with_flags[:-1], without[:-1])):
        assert (np.where(s1 == M.CORRUPT, M.HIT, s1) == s2).all(), (k, s1, s2)
        for i, page in p1.items():
            assert p2[i] == page, (k, i)


@pytest.mark.parametrize("pshift", [16, 17])
def test_a_small_get_waits_for_its_lanes_previous_probe(E, gpu, oracle, tmp_path, monkeypatch, pshift):
    """The script's lane step with 1024 turns: a begin that takes the lane the other thread has just freed finds
    that get's ghost probe still running often enough that cmb200_get_small_begin waits for it
    (lane_waits), and the table, the statuses and the pages stay the model's.  No FREQ: so many gets in one
    step would cross a halving, and the threads' order would then decide the sketch."""
    case = dict(id=f"p{pshift}-VTG-lanes", pshift=pshift, flags=M.VERIFY | M.TOUCH | M.GHOST, ckpt0=False)
    _, waits = _run(E, case, case["flags"], tmp_path, monkeypatch, lane_reps=1024)
    print(f"{case['id']}: lane waits {waits}")
    assert waits > 0


@pytest.mark.parametrize("pshift", [16, 17])
@pytest.mark.parametrize("verify,touch,freq", [(v, t, f) for v in (0, 1) for t in (0, 1) for f in (0, 1)],
                         ids=lambda b: str(b))
def test_every_fused_get_variant_at_full_occupancy(E, gpu, oracle, tmp_path, pshift, verify, touch, freq):
    """One cmb200_get_small of 1 024 distinct compressed records: more requests than the device holds CTAs,
    so scratch regions are handed on within the launch.  Every answer is HIT with its exact page, and the
    counters are the model's."""
    n, bs = 1024, 1 << pshift
    flags = (M.VERIFY if verify else 0) | (M.TOUCH if touch else 0) | (M.FREQ if freq else 0)
    e = E.Engine(pshift=pshift, capacity=n, arena_bytes=512 << 20, max_batch=256, flags=flags)
    try:
        rng = random.Random(pshift)
        addrs = [(31 + k % 3, k) for k in range(n)]
        rng.shuffle(addrs)
        pages = np.stack([M.page_of(a, 1, bs) for a in addrs])
        lens = e.put(*_arrays(addrs), pages, ts=np.arange(1, n + 1, dtype=np.uint64))
        assert (lens > 0).all()                                   # every record is an LZ4 block
        buf = _Pinned(E, n, bs)
        try:
            st = np.zeros(n, dtype=np.int32)
            t0 = coarse_ns()
            addr = _addr(addrs)
            assert E.lib().cmb200_get_small(e.h, n, addr.ctypes.data, buf.p, st.ctypes.data) == 0
            t1 = coarse_ns()
            assert (st == M.HIT).all(), np.unique(st, return_counts=True)
            assert (buf.pages() == pages).all()
        finally:
            buf.free()
        vs = e.verify_stats()
        assert (vs["verified"], vs["unverified"], vs["corrupt"]) == ((n, 0, 0) if verify else (0, 0, 0)), vs
        if freq:
            sk = A.Sketch(n)
            sk.launch([A.fnv_addr(*a) for a in addrs])
            assert (e.freq_read() == sk.words()).all()
            assert e.freq_stats()["increments"] == n
        got_ts = _ts_all(e, str(tmp_path / "ts.snap"))
        for k, a in enumerate(addrs):
            if touch:
                assert t0 <= got_ts[a] <= t1, (a, got_ts[a], t0, t1)
            else:
                assert got_ts[a] == k + 1, a
    finally:
        e.close()
