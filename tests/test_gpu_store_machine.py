"""One engine driven through long seeded interleavings of every engine operation, compared after every
step with the model of tests/store_machine.py: entries, every record byte, fingerprints, parse
checkpoints, get answers on both get paths, arena and host-tier accounting, verification counters,
sampled addresses and timestamps, and the request counters.  A failure names its configuration, seed
and step and prints the log of the operations that led there."""
import ctypes as C
import time

import numpy as np
import pytest

import store_machine as SM

pytestmark = pytest.mark.gpu

# the touch stamp is read from CLOCK_REALTIME_COARSE, which lags CLOCK_REALTIME by up to a tick
COARSE_SLACK_NS = 20_000_000


def _addr(addrs):
    u = np.array([a[0] for a in addrs], dtype=np.uint64)
    l = np.array([a[1] for a in addrs], dtype=np.uint64)
    return u, l


class Machine:
    def __init__(self, E, oracle, cfg, seed, tmp_path):
        self.E, self.O, self.cfg, self.seed, self.tmp = E, oracle, cfg, seed, tmp_path
        self.m = SM.Model(cfg, oracle)
        self.eng = self._engine(cfg.table_slots, cfg.arena_bytes)
        self.U = list(dict.fromkeys(SM.universe(cfg)))
        self.Uu, self.Ul = _addr(self.U)
        self.log = []

    def _engine(self, slots, arena):
        c = self.cfg
        return self.E.Engine(pshift=c.pshift, accel=c.accel, capacity=slots // 4, arena_bytes=arena,
                             table_slots=slots, max_batch=c.max_batch, flags=c.flags,
                             host_tier_bytes=c.tier_bytes)

    def run(self):
        for step, op in enumerate(SM.gen_ops(self.cfg, self.seed)):
            self.log.append(f"{step:4d} {SM.describe(op)}")
            try:
                getattr(self, "op_" + op[0])(op, step)
                self.check(op[0])
            except AssertionError as e:
                raise AssertionError(f"config {self.cfg.name} seed {self.seed} step {step} ({op[0]}): {e}\n"
                                     "op log (replay: store_machine.gen_ops(CONFIGS[config], seed)):\n"
                                     + "\n".join(self.log[-60:])) from None
        self.eng.close()

    # ---- operations
    def _put(self, op, lens_of):
        _, addrs, specs, ts, valid = op
        pages = SM.pages_of(self.cfg, specs)
        u, l = _addr(addrs)
        tsa = None if ts is None else np.array(ts, dtype=np.uint64)
        va = None if valid is None else np.array(valid, dtype=np.uint8)
        must_drop = self.m.cfg.exact_head and self.m.certain_drop(addrs, pages, valid)
        lens = lens_of(u, l, pages, tsa, va)
        rows = self.m.put_rows(addrs, valid)
        skipped = sorted(set(range(len(addrs))) - set(rows))
        assert (lens[skipped] == -1).all(), f"lens of superseded or invalid rows: {lens[skipped].tolist()}"
        dropped = {i for i in rows if lens[i] == -1}
        for i in rows:
            if i not in dropped:
                want = self.m.make(addrs[i], pages[i], 0).clen
                assert lens[i] == want, f"row {i}: lens {lens[i]}, stored block {want}"
        if self.m.cfg.exact_head:
            assert bool(dropped) == must_drop, f"drops {sorted(dropped)}; the arena certainly overflows: {must_drop}"
        self.m.put(addrs, pages, ts, valid, dropped)

    def op_put(self, op, step):
        self._put(op, lambda u, l, p, ts, v: self.eng.put(u, l, p, ts=ts, valid=v))

    def op_put_async(self, op, step):
        def go(u, l, p, ts, v):
            n = len(u)
            buf = self.E.lib().cmb200_host_alloc(4 * n)
            try:
                t = self.eng.put_async(u, l, p, ts=ts, valid=v, lens=buf)
                self.eng.wait(t)
                return np.ctypeslib.as_array((C.c_int32 * n).from_address(buf)).copy()
            finally:
                self.E.lib().cmb200_host_free(buf)
        self._put(op, go)

    def _get(self, addrs, got, status, valid, t0, t1):
        exp = self.m.get(addrs, valid, t0 - COARSE_SLACK_NS, t1)
        for i, (st, pg) in enumerate(exp):
            assert status[i] == st, f"get row {i} {addrs[i]}: status {status[i]}, model {st}"
            if st == SM.HIT:
                assert got[i].tobytes() == pg, f"get row {i} {addrs[i]}: page differs"

    def op_get(self, op, step):
        _, addrs, valid = op
        u, l = _addr(addrs)
        t0 = time.clock_gettime_ns(time.CLOCK_REALTIME)
        out, status = self.eng.get(u, l, valid=None if valid is None else np.array(valid, dtype=np.uint8))
        t1 = time.clock_gettime_ns(time.CLOCK_REALTIME)
        self._get(addrs, out, status, valid, t0, t1)

    def op_get_small(self, op, step):
        _, addrs, _ = op
        u, l = _addr(addrs)
        t0 = time.clock_gettime_ns(time.CLOCK_REALTIME)
        out, status = self.eng.get_small(u, l)
        t1 = time.clock_gettime_ns(time.CLOCK_REALTIME)
        self._get(addrs, out, status, None, t0, t1)

    def op_unset(self, op, step):
        self.eng.unset(*_addr(op[1]))
        self.m.unset(op[1])

    def op_invalidate(self, op, step):
        _, u, lf, ll = op
        got = self.eng.invalidate(u, lf, ll)
        want = self.m.invalidate(u, lf, ll)
        self.m.rebuild_check()
        assert got == want, f"invalidate removed {got}, model {want}"

    def op_compact(self, op, step):
        self.eng.compact()
        self.m.compact()
        self.m.rebuild_check()
        st = self.eng.stats()
        assert st["arena_garbage"] == 0, st["arena_garbage"]
        assert st["arena_used"] == self.m.arena_alloc(), (st["arena_used"], self.m.arena_alloc())

    def op_demote(self, op, step):
        got = self.eng.demote(*_addr(op[1]))
        want, _ = self.m.demote(op[1])
        assert got == want, f"demoted {got}, model {want}"

    def op_promote(self, op, step):
        got = self.eng.promote(*_addr(op[1]))
        want = self.m.promote(op[1])
        assert got == want, f"promoted {got}, model {want}"

    def op_sample(self, op, step):
        addr, ts, ok = self.eng.sample(np.array(op[1], dtype=np.uint64))
        for i in range(len(op[1])):
            if ok[i] == 0:
                assert not self.m.rec, f"sample {i}: none found, model holds {len(self.m.rec)}"
                continue
            assert ok[i] == 1, ok[i]
            a = (int(addr[i, 0]), int(addr[i, 1]))
            r = self.m.live(a)
            assert r is not None, f"sample {i}: {a} holds no record"
            assert r.ts_lo <= int(ts[i]) <= r.ts_hi, f"sample {i} {a}: ts {int(ts[i])} outside [{r.ts_lo}, {r.ts_hi}]"
            r.ts_lo = r.ts_hi = int(ts[i])

    def op_verify_store(self, op, step):
        _, _, bad, checked = self.eng.verify_store()
        assert bad == 0 and checked == self.m.fp_records(), (bad, checked, self.m.fp_records())

    def op_load(self, op, step):
        path = str(self.tmp / f"snap.{self.cfg.name}.{self.seed}")
        assert self.eng.save(path) == len(self.m.rec)
        fresh = self._engine(self.cfg.load_slots, self.cfg.load_arena)
        try:
            assert fresh.load(path) == len(self.m.rec)
        except BaseException:
            fresh.close()
            raise
        self.eng.close()
        self.eng = fresh
        self.m.load(self.cfg.load_slots, self.cfg.load_arena)

    # ---- after every step
    def check(self, kind):
        m, eng, cfg = self.m, self.eng, self.cfg
        st = eng.stats()
        assert st["entries"] == len(m.rec), f"entries {st['entries']}, model {len(m.rec)}"
        assert st["dropped_puts"] == m.ctr.dropped, f"dropped_puts {st['dropped_puts']}, model {m.ctr.dropped}"
        assert (st["get_requests"], st["get_hits"]) == (m.ctr.requests, m.ctr.hits), \
            f"requests / hits {(st['get_requests'], st['get_hits'])}, model {(m.ctr.requests, m.ctr.hits)}"
        live = [m.live(a) for a in self.U]
        recs = eng.read_records(self.Uu, self.Ul)
        for a, r, got in zip(self.U, live, recs):
            want = None if r is None else self.O.record_prefix(a[0], a[1], r.clen) + r.block
            assert got == want, f"record of {a}: {'absent' if got is None else len(got)} bytes, model " \
                                f"{'absent' if want is None else len(want)} bytes{' (bytes differ)' if got and want else ''}"
        if cfg.flags & (SM.FINGERPRINT | SM.VERIFY):
            fps, ok = eng.read_fingerprints(self.Uu, self.Ul)
            for i, (a, r) in enumerate(zip(self.U, live)):
                assert bool(ok[i]) == (r is not None), f"fingerprint of {a}: ok {ok[i]}"
                if r is not None and r.has_fp:
                    assert (int(fps[i, 0]), int(fps[i, 1])) == r.fp, f"fingerprint of {a} differs"
        words, ok = eng.read_checkpoints(self.Uu, self.Ul)
        ckpt_on = cfg.environ().get("CMB200_CKPT") != "0"
        for i, (a, r) in enumerate(zip(self.U, live)):
            if not ckpt_on or r is None:
                assert ok[i] == -1, f"checkpoints of {a}: ok {ok[i]}, want -1"
            elif r.ckpt is None:
                assert ok[i] == 0, f"checkpoints of {a} (raw or unwalkable block): ok {ok[i]}, want 0"
            else:
                assert ok[i] == 1 and words[i, 1:].tolist() == r.ckpt[1:], \
                    f"checkpoints of {a}: ok {ok[i]}, words {'equal' if words[i, 1:].tolist() == r.ckpt[1:] else 'differ'}"
        if cfg.exact_head and not m.saturated:
            assert st["arena_used"] == m.head, f"arena_used {st['arena_used']}, model bump pointer {m.head}"
            assert st["arena_used"] == m.arena_alloc() + st["arena_garbage"], \
                f"arena_used {st['arena_used']} != alloc {m.arena_alloc()} + garbage {st['arena_garbage']}"
        if cfg.tier_bytes:
            ht = eng.host_tier_stats()
            want = {"records": m.tier_records(), "used": m.tier_used(), "garbage": m.tier_garbage(),
                    "retired_records": m.ctr.retired}
            got = {k: ht[k] for k in want}
            assert got == want, f"host tier {got}, model {want}"
        if cfg.flags & SM.VERIFY:
            vs = eng.verify_stats()
            got = (vs["verified"], vs["unverified"], vs["corrupt"])
            assert got == (m.ctr.verified, m.ctr.unverified, 0), f"verify counters {got}, model {(m.ctr.verified, m.ctr.unverified, 0)}"


@pytest.fixture
def machine_env(monkeypatch):
    def setup(cfg):
        for k in ("CMB200_SEG_KB", "CMB200_CKPT"):
            monkeypatch.delenv(k, raising=False)
        for k, v in cfg.env:
            monkeypatch.setenv(k, v)
    return setup


@pytest.mark.parametrize("name,seed", [(n, s) for n in sorted(SM.CONFIGS) for s in SM.CONFIGS[n].seeds])
def test_store_machine(E, gpu, oracle, tmp_path, machine_env, name, seed):
    cfg = SM.CONFIGS[name]
    machine_env(cfg)
    Machine(E, oracle, cfg, seed, tmp_path).run()


def test_dropped_put_reports_minus_one(E, gpu, monkeypatch):
    """A put the full arena drops stored nothing: its lens entry is -1, as for a skipped chunk, and the
    key keeps serving its old record."""
    monkeypatch.setenv("CMB200_SEG_KB", "0")
    import datagen
    eng = E.Engine(pshift=12, accel=12, capacity=256, arena_bytes=64 << 10, max_batch=64)
    u = np.full(32, 4, dtype=np.uint64)
    l = np.arange(32, dtype=np.uint64)
    small = np.stack([datagen.make_page("Z", 4096, i) for i in range(32)])
    assert (eng.put(u, l, small) > 0).all()
    big = np.stack([datagen.make_page("R", 4096, 100 + i) for i in range(32)])   # ~4.1 KiB records: half fit
    lens = eng.put(u, l, big)
    out, status = eng.get(u, l)
    assert (status == E.HIT).all()
    new = np.array([(out[i] == big[i]).all() for i in range(32)])
    assert 0 < new.sum() < 32 and all((out[i] == small[i]).all() for i in np.nonzero(~new)[0])
    assert (lens[~new] == -1).all() and (lens[new] > 4096).all(), lens.tolist()
    assert eng.stats()["dropped_puts"] == int((~new).sum())
    eng.close()
