"""GPU tests of reads from another rank's arena (ST_REMOTE in k_get_small and k_get_small_pair) on one
device.  Two child processes (tests/peer_owner.py) play ranks 0 and 2: each owns an engine, stores its
shard with put_step and exports its arena by CUDA IPC.  This process is rank 1: it imports the children's
exchange records, maps their arenas with open_peer and reads through the same kernel code a multi-GPU
run uses; only the transport differs (local HBM instead of NVLink).  Every expected page comes from the
generator, never from another get path.

Lifetime: a get is only issued against children whose last command was answered; the peers are closed
(close_peers) before a child frees its engine; each child exits with code 0 at the end of the module."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import datagen
import key_edges
from edge_fuse_b200 import sharding
from test_gpu_get_small_128k import _pages as pages_128k

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEER_OWNER = os.path.join(ROOT, "tests", "peer_owner.py")
KINDS = "RTZMPAX"
WORLD, ME = 3, 1                                 # children are ranks 0 and 2
ARENA = 48 << 20


class Child:
    """A rank in a child process: one JSON command per line (tests/peer_owner.py)."""

    def __init__(self, rank, tmp):
        self.rank, self.dir, self.k = rank, str(tmp), 0
        self.p = subprocess.Popen([sys.executable, PEER_OWNER], cwd=ROOT, stdin=subprocess.PIPE,
                                  stdout=subprocess.PIPE, text=True)
        self.open = False

    def npy(self, a):
        self.k += 1
        path = os.path.join(self.dir, f"in{self.k}.npy")
        np.save(path, np.ascontiguousarray(a))
        return path

    def call(self, cmd, **kw):
        self.p.stdin.write(json.dumps({"cmd": cmd, "dir": self.dir, **kw}) + "\n")
        self.p.stdin.flush()
        line = self.p.stdout.readline()
        assert line, f"rank {self.rank} exited during {cmd}"
        ans = json.loads(line)
        assert ans["ok"], f"rank {self.rank} {cmd}: {ans['error']}"
        return ans

    def finish(self):
        try:
            self.p.stdin.close()
        except OSError:
            pass
        try:
            self.p.wait(timeout=60)
        except subprocess.TimeoutExpired:
            self.p.kill()
            self.p.wait()
        return self.p.returncode


@pytest.fixture(scope="module")
def kids(E, gpu, tmp_path_factory):
    t0 = time.time()
    card = "unknown card"
    try:                                         # a read-only query: name and power limit of the card
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or card
    except (OSError, subprocess.SubprocessError):
        pass
    print(f"\n[peer reads] {card}")
    ks = {r: Child(r, tmp_path_factory.mktemp(f"rank{r}")) for r in (0, 2)}
    try:
        yield ks
    finally:
        codes = {r: k.finish() for r, k in ks.items()}
        print(f"\n[peer reads] file wall time {time.time() - t0:.1f} s")
    assert codes == {0: 0, 2: 0}, codes


class World:
    """Rank 1 (this process's engine) and the two children, at one page size."""

    def __init__(self, E, kids, pshift):
        self.E, self.kids, self.pshift, self.bs = E, kids, pshift, 1 << pshift
        self.eng = None
        self.base = 1000
        self.pages = {}                          # (u, l) -> every page ever stored there
        self.want = {}                           # (u, l) -> (status seen by rank 1, page or None, owner)

    def start(self, accel, flags):
        for k in self.kids.values():
            k.call("create", pshift=self.pshift, accel=accel, flags=0, arena_bytes=ARENA, capacity=1024)
            k.open = True
        # rank 1's arena is smaller than the offsets it reads from its peers: each child first stores
        # ballast it never exports, so a bound taken from the reader's own arena turns remote hits into misses
        self.arena = max(64 << 10, 32 * (self.bs + 1088))
        self.eng = self.E.Engine(pshift=self.pshift, accel=accel, capacity=1024, arena_bytes=self.arena,
                                 max_batch=256, flags=flags)
        nb = self.arena // self.bs + 2
        for k in self.kids.values():
            k.call("put", u_npy=k.npy(np.full(nb, 0xBA11, np.uint64)), l_npy=k.npy(np.arange(nb, dtype=np.uint64)),
                   pages={"gen": [["R", 77 + i] for i in range(nb)]})

    def close(self):
        if self.eng is not None:
            self.eng.close_peers()               # no mapping outlives the arena behind it
        for k in self.kids.values():
            if k.open:
                k.call("close")
                k.open = False
        if self.eng is not None:
            self.eng.close()
            self.eng = None

    def step(self, shards, valid=None):
        """One put step: shards = {rank: (u, l, pages)}.  -> all-gathered [n, 4] rows (rank 1's own included)."""
        rows = []
        for r, (u, l, pages) in sorted(shards.items()):
            v = np.ones(len(u), np.uint8) if valid is None or r not in valid else valid[r]
            if r == ME:
                d = self.eng.dev_alloc(len(u) * 32)
                self.eng.set_stream_order(self.base + r, WORLD)
                self.eng.wait(self.eng.put_step(u, l, pages, valid=v, rank=r, records_dev=d))
                self.eng.sync()
                rec = np.zeros((len(u), 4), np.int64)
                self.eng.d2h(rec, d)
                self.eng.dev_free(d)
            else:
                k = self.kids[r]
                ans = k.call("put_step", u_npy=k.npy(u), l_npy=k.npy(l), valid_npy=k.npy(v),
                             pages={"npy": k.npy(pages)}, rank=r, base=self.base + r, stride=WORLD)
                rec = np.load(ans["records_npy"])
            rows.append(rec)
            for i in range(len(u)):
                if v[i]:
                    key = (int(u[i]), int(l[i]))
                    self.pages.setdefault(key, []).append(pages[i])
                    self.want[key] = (self.E.HIT if r == ME else self.E.REMOTE, pages[i], r)
        self.base += WORLD * max(len(s[0]) for s in shards.values())
        return np.concatenate(rows)

    def import_rows(self, rows):
        d = self.eng.dev_alloc(rows.nbytes)
        try:
            self.eng.h2d(d, np.ascontiguousarray(rows))
            self.eng.import_records_dev(len(rows), d, ME)
            self.eng.sync()
        finally:
            self.eng.dev_free(d)

    def open_peers(self):
        for r, k in self.kids.items():
            h = k.call("handle")
            self.eng.open_peer(r, bytes.fromhex(h["handle"]), h["size"])

    def locate(self, r, u, l):
        k = self.kids[r]
        a = k.call("locate", u_npy=k.npy(u), l_npy=k.npy(l))
        return np.load(a["status_npy"]), np.load(a["where_npy"]).astype(np.uint64), np.load(a["clen_npy"])


@pytest.fixture
def world(E, kids):
    made = []

    def make(pshift, accel, flags=0):
        w = World(E, kids, pshift)
        made.append(w)
        w.start(accel, flags)
        return w
    try:
        yield make
    finally:
        for w in made:
            w.close()


def shard_pages(pshift, n, seed):
    bs = 1 << pshift
    return np.stack([datagen.make_page(KINDS[i % len(KINDS)], bs, seed + i) for i in range(n)])


def addrs(u0, n):
    return np.full(n, u0, np.uint64), np.arange(n, dtype=np.uint64)


def standard_world(make, pshift, accel, n=28, flags=0, open_peers=True):
    """Each child stores n pages of every datagen class (at 128 KiB rank 0's first three are the wide
    descriptor pages of test_gpu_get_small_128k), rank 1 stores 16; rank 0 also stores one address of a
    key-sharing pair and rank 1 one of another; one address of each child's step is invalid."""
    w = make(pshift, accel, flags)
    fx = key_edges.load()
    shards = {}
    for r in (0, 1, 2):
        m = n if r != ME else 16
        u, l = addrs(0xA000 + r, m)
        pages = shard_pages(pshift, m, 1000 * r + 37 * pshift + accel)
        if pshift == 17 and r == 0:
            pages[:3] = pages_128k(3, 4242)
        if r != ME:
            u[-1], l[-1] = fx["groups"]["pair0" if r == 0 else "pair2"][0]
        else:
            u[-1], l[-1] = fx["groups"]["pair1"][0]
        shards[r] = (u, l, pages)
    valid = {0: np.ones(n, np.uint8), 2: np.ones(n, np.uint8)}
    valid[0][5] = 0
    valid[2][9] = 0
    rows = w.step(shards, valid)
    w.import_rows(rows)
    if open_peers:
        w.open_peers()
    w.shards = shards
    w.sharing = {"remote": fx["groups"]["pair0"][1], "local": fx["groups"]["pair1"][1]}
    return w, rows


def expected(w, keys):
    """-> status, pages (zeros where no page), owner of each (u, l) as rank 1's get_small answers it with
    the peers open.  The other address of a key rank 1 stores answers BAD_ENTRY; the other address of a key
    whose newest record is on a peer answers MISS (DESIGN.md §9)."""
    E = w.E
    st = np.full(len(keys), E.MISS, np.int32)
    pg = np.zeros((len(keys), w.bs), np.uint8)
    ow = np.full(len(keys), -1)
    for i, k in enumerate(keys):
        if k in w.want:
            s, p, r = w.want[k]
            st[i] = E.HIT
            pg[i] = p
            ow[i] = r
        elif k == tuple(w.sharing["local"]):
            st[i] = E.BAD_ENTRY
    return st, pg, ow


def query_keys(w):
    keys = [k for k in w.want]
    keys += [(0xB000, i) for i in range(5)]                     # never stored
    keys += [(0xA000, 5), (0xA002, 9)]                          # invalid in their step: stored nothing
    keys += [tuple(w.sharing["remote"]), tuple(w.sharing["local"])]
    return keys


def split(keys):
    return (np.array([k[0] for k in keys], np.uint64), np.array([k[1] for k in keys], np.uint64))


def check_small(w, keys, what=""):
    u, l = split(keys)
    out, st = w.eng.get_small(u, l)
    want_st, want_pg, _ = expected(w, keys)
    bad = np.nonzero(st != want_st)[0]
    assert len(bad) == 0, (what, w.pshift, [(keys[i], int(st[i]), int(want_st[i])) for i in bad[:8]])
    hit = want_st == w.E.HIT
    rows = np.nonzero(hit & (out != want_pg).any(axis=1))[0]
    assert len(rows) == 0, (what, w.pshift, [keys[i] for i in rows[:8]])
    return st


@pytest.mark.parametrize("accel", [12, 0], ids=["lz4", "raw"])
@pytest.mark.parametrize("pshift", list(range(6, 18)))
def test_every_fused_get_page_size(E, world, pshift, accel):
    """A: remote keys mixed with local keys, misses and key-sharing addresses in one call: each answer is
    the right status and the exact page; the batch get answers REMOTE and locate names the owner."""
    w, _ = standard_world(world, pshift, accel)
    keys = query_keys(w)
    check_small(w, keys)
    u, l = split(keys)
    want_st, want_pg, want_ow = expected(w, keys)
    remote = want_ow >= 0
    remote &= np.array([w.want.get(k, (0, 0, ME))[2] != ME for k in keys])
    assert remote.sum() == 2 * 27
    out, st = w.eng.get(u, l)
    assert (st[remote] == E.REMOTE).all()
    assert (st[~remote] == want_st[~remote]).all()
    local = ~remote & (want_st == E.HIT)
    assert (out[local] == want_pg[local]).all()
    s2, o2 = w.eng.locate(u, l)
    assert (s2[remote] == E.REMOTE).all() and (o2[remote] == want_ow[remote].astype(np.uint64)).all()
    assert w.eng.stats()["remote_entries"] == 2 * 27
    # full calls, about half remote: lanes and scratch regions are reused across calls
    rng = np.random.default_rng(pshift * 7 + accel)
    rem = [k for k, i in zip(keys, remote) if i]
    rest = [k for k, i in zip(keys, remote) if not i]
    for call in range(3):
        pick = [rem[int(j)] for j in rng.integers(0, len(rem), 512)] + \
               [rest[int(j)] for j in rng.integers(0, len(rest), 512)]
        pick = [pick[int(j)] for j in rng.permutation(1024)]
        check_small(w, pick, f"call {call}")


@pytest.mark.parametrize("pshift,accel", [(12, 0), (16, 12), (17, 12)])
def test_stale_locations(E, world, pshift, accel):
    """B: rank 0 rewrites and unsets keys without exporting: rank 1 serves the imported version (the bytes
    stay until compaction).  After rank 0 compacts, every answer is a miss or a page rank 0 stored at that
    address, and a record that did not move is a hit.  Rows from rank 0's current locations at a higher
    position make every live key a hit again."""
    w, rows = standard_world(world, pshift, accel)
    keys = query_keys(w)
    check_small(w, keys, "fresh")
    u0, l0, pages0 = w.shards[0]
    n = len(u0)
    rewr = np.arange(n - 12, n - 6)                   # rewritten
    gone = np.arange(n - 6, n)                        # removed (the last is the key-sharing address)
    new = shard_pages(pshift, len(rewr), 5555 + pshift)
    k0 = w.kids[0]
    k0.call("put", u_npy=k0.npy(u0[rewr]), l_npy=k0.npy(l0[rewr]), pages={"npy": k0.npy(new)})
    k0.call("unset", u_npy=k0.npy(u0[gone]), l_npy=k0.npy(l0[gone]))
    check_small(w, keys, "after rewrite and unset")   # still the imported version of every key
    for j, i in enumerate(rewr):
        w.pages[(int(u0[i]), int(l0[i]))].append(new[j])
    assert k0.call("compact")["reclaimed"] > 0
    imp_u, imp_l, _, imp_owner, imp_len = sharding.unpack_records(rows)
    imp_off = sharding.unpack_locations(rows).astype(np.uint64)
    imported = {}
    for i in range(len(rows)):
        if imp_owner[i] == 0 and imp_len[i] >= 0:
            imported[(int(np.uint64(imp_u[i])), int(np.uint64(imp_l[i])))] = (int(imp_off[i]), int(imp_len[i]))
    st0, where, clen = w.locate(0, u0, l0)
    cur = {}
    for i in range(n):
        if st0[i] == E.HIT:
            cur[(int(u0[i]), int(l0[i]))] = (int(where[i]), int(clen[i]))
    ru, rl = split(list(imported))
    out, st = w.eng.get_small(ru, rl)
    same = 0
    for i, k in enumerate(imported):
        assert st[i] in (E.MISS, E.HIT), (k, st[i])
        if st[i] == E.HIT:
            assert any((out[i] == p).all() for p in w.pages[k]), k
        if cur.get(k) == imported[k]:
            same += 1
            assert st[i] == E.HIT, (k, "record did not move")
    assert same < len(imported)                       # some imported locations are stale now
    # rank 0's current locations, at a position above every row so far
    live = list(cur)
    lu, ll = split(live)
    fresh = sharding.pack_records(lu, ll, np.full(len(live), w.base + 10_000, np.uint64), 0,
                                  [cur[k][1] for k in live], [cur[k][0] for k in live])
    w.import_rows(fresh)
    out, st = w.eng.get_small(lu, ll)
    assert (st == E.HIT).all(), [(live[i], int(st[i])) for i in np.nonzero(st != E.HIT)[0][:8]]
    for i, k in enumerate(live):
        assert (out[i] == w.pages[k][-1]).all(), k
    print(f"\n[stale {pshift}] {same} of {len(imported)} records kept their place")


@pytest.mark.parametrize("accel", [12, 0], ids=["lz4", "raw"])
def test_locations_that_do_not_name_the_record(E, world, accel):
    """C: imported rows that point 16 bytes into a record, at another address's record, or at the right
    record with a length other than the prefix's compressed_length: MISS, never a page.  Every forged
    offset lies below rank 0's arena_used."""
    w, _ = standard_world(world, 12, accel)
    u0, l0, _ = w.shards[0]
    st0, where, clen = w.locate(0, u0, l0)
    used = w.kids[0].call("stats")["arena_used"]
    ok = np.nonzero(st0 == E.HIT)[0]
    order = ok[np.argsort(where[ok])]
    assert len(order) >= 10
    fu, fl, fo, fn = [], [], [], []

    def forge(i, off, ln):
        assert off < used and off % 16 == 0
        fu.append(u0[i]); fl.append(l0[i]); fo.append(off); fn.append(ln)
    forge(order[0], int(where[order[0]]) + 16, int(clen[order[0]]))           # 16 bytes into its own record
    forge(order[1], int(where[order[2]]), int(clen[order[2]]))                # another address's record
    forge(order[3], int(where[order[4]]), int(clen[order[3]]))
    for j, i in enumerate(order[5:9]):                                        # right place, wrong length
        c = int(clen[i])
        alt = [c + 16, c - 1, 0, c + 1][j] if c > 0 else [1, 16, w.bs, w.bs - 24][j]
        assert alt != c and alt >= 0
        forge(i, int(where[i]), alt)
    rows = sharding.pack_records(fu, fl, np.full(len(fu), w.base + 50, np.uint64), 0, fn, fo)
    w.import_rows(rows)
    if accel == 0:
        assert (clen[order[:9]] == 0).all()
    else:
        assert (clen[order[:9]] > 0).all()
    forged = {(int(a), int(b)) for a, b in zip(fu, fl)}
    for k in forged:
        w.want[k] = (E.MISS, None, 0)
    keys = query_keys(w)
    u, l = split(keys)
    out, st = w.eng.get_small(u, l)
    for i, k in enumerate(keys):
        if k in forged:
            assert st[i] == E.MISS, (k, int(st[i]))
    for k in forged:
        del w.want[k]
    check_small(w, [k for k in keys if k not in forged], "the rest")


@pytest.mark.parametrize("pshift", [16, 17])
def test_no_mapping(E, world, pshift):
    """D: REMOTE, never a fault, before open_peer, after close_peers, for an owner rank with no peer open
    and for owner ranks >= GET_MAX_PEERS (16); the same keys are hits once the peers are open again."""
    w, _ = standard_world(world, pshift, 12, n=20, open_peers=False)
    keys = query_keys(w)
    u, l = split(keys)
    want_st, want_pg, want_ow = expected(w, keys)
    remote = np.array([w.want.get(k, (0, 0, ME))[2] != ME for k in keys])

    def answers(peers_open):
        out, st = w.eng.get_small(u, l)
        exp = want_st.copy()
        if not peers_open:
            exp[remote] = E.REMOTE
        for i, k in enumerate(keys):
            if k in odd:
                exp[i] = E.REMOTE
        bad = np.nonzero(st != exp)[0]
        assert len(bad) == 0, [(keys[i], int(st[i]), int(exp[i])) for i in bad[:8]]
        hit = exp == E.HIT
        assert (out[hit] == want_pg[hit]).all()

    odd = set()
    answers(False)                                          # before open_peer
    # rank 2's real locations, claimed by ranks with no mapping: 5 (none opened), 16 and 200 (out of range)
    u2, l2, _ = w.shards[2]
    st2, where, clen = w.locate(2, u2, l2)
    idx = np.nonzero(st2 == E.HIT)[0][:6]
    rows = np.concatenate([sharding.pack_records(u2[idx[2 * j:2 * j + 2]], l2[idx[2 * j:2 * j + 2]],
                                                 np.full(2, w.base + 100 + j, np.uint64), r,
                                                 clen[idx[2 * j:2 * j + 2]], where[idx[2 * j:2 * j + 2]])
                           for j, r in enumerate((5, 16, 200))])
    w.import_rows(rows)
    odd = {(int(u2[i]), int(l2[i])) for i in idx}
    s2, o2 = w.eng.locate(u2[idx], l2[idx])
    assert (s2 == E.REMOTE).all() and list(o2) == [5, 5, 16, 16, 200, 200]
    answers(False)
    w.open_peers()
    answers(True)
    w.eng.close_peers()
    answers(False)                                          # after close_peers
    w.open_peers()
    answers(True)


@pytest.mark.parametrize("pshift", [16, 17])
def test_flags_on_the_reading_engine(E, world, pshift):
    """E: with VERIFY every remote hit counts as unverified and none is CORRUPT; with FINGERPRINT alone
    the remote keys have no fingerprint."""
    w, _ = standard_world(world, pshift, 12, flags=E.VERIFY)
    keys = query_keys(w)
    want_st, _, _ = expected(w, keys)
    remote = np.array([w.want.get(k, (0, 0, ME))[2] != ME for k in keys])
    v0 = w.eng.verify_stats()
    st = check_small(w, keys, "verify")
    v1 = w.eng.verify_stats()
    assert v1["corrupt"] == v0["corrupt"]
    assert v1["unverified"] - v0["unverified"] == int(remote.sum())
    assert v1["verified"] - v0["verified"] == int(((st == E.HIT) & ~remote).sum())
    w.close()                                         # each child holds one engine at a time
    w, _ = standard_world(world, pshift, 12, flags=E.FINGERPRINT)
    check_small(w, keys, "fingerprint")
    u, l = split(keys)
    _, ok = w.eng.read_fingerprints(u, l)
    assert (ok[remote] == 0).all() and (ok[(want_st == E.HIT) & ~remote] == 1).all()


# ---- the replicated index against its sequential model (tests/replica_model.py) -----------------------

def _model_check(E, engs, models, used, what):
    """Every engine against its model: locate status and owner of every address used so far, entries and
    remote_entries, the pages of local hits, and sample never naming a remote address."""
    addrs = sorted(used)
    u, l = split(addrs)
    for r, (eng, m) in enumerate(zip(engs, models)):
        st, ow = eng.locate(u, l)
        want = [m.lookup(a) for a in addrs]
        bad = [(addrs[i], int(st[i]), want[i][:2]) for i in range(len(addrs))
               if st[i] != want[i][0] or (want[i][0] == E.REMOTE and int(ow[i]) != want[i][1])]
        assert not bad, (what, r, bad[:6])
        s = eng.stats()
        assert (s["entries"], s["remote_entries"]) == (m.entries(), m.remote_entries()), (what, r)
        hits = [i for i in range(len(addrs)) if want[i][0] == E.HIT]
        if hits:
            out, gst = eng.get(u[hits], l[hits])
            assert (gst == E.HIT).all(), (what, r)
            for j, i in enumerate(hits):
                assert (out[j] == want[i][2]).all(), (what, r, addrs[i])
        sa, _, ok = eng.sample(np.arange(64, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        local = m.local_records()
        for j in np.nonzero(ok)[0]:
            assert (int(sa[j, 0]), int(sa[j, 1])) in local, (what, r, sa[j])


@pytest.mark.parametrize("seed", range(4))
def test_replicated_index_against_the_sequential_model(E, gpu, tmp_path, seed):
    """Three engines on one device play ranks 0..2 at pshift 12; the all-gather is done on the host.
    Steps with repeated, invalid, duplicated, key-sharing and sentinel addresses and puts the arena drops;
    rows imported 0 to 2 steps late in shuffled order; between steps, on a random engine: a put below an
    imported row of the same key, unsets of local and remote keys, compaction, a table rebuild, save and
    load into a fresh engine, verify_store.  After every operation every engine answers as its model."""
    import replica_model as RM
    rng = np.random.default_rng(1234 + seed)
    fx = key_edges.load()
    bs, world = 1 << 12, 3
    pool = [(0xC000 + int(i % 3), int(i)) for i in range(150)]
    pool += [a for g in ("quad", "pair0", "pair1", "key0", "key_ones") for a in fx["groups"][g]]
    engs = [E.Engine(pshift=12, accel=12, table_slots=512, arena_bytes=(256 << 10) if r == 2 else (32 << 20),
                     max_batch=64, flags=E.VERIFY) for r in range(world)]
    models = [RM.ReplicaModel(r) for r in range(world)]
    d_rec = [e.dev_alloc(64 * 32) for e in engs]
    used, pending, pos, pid = set(), [], 1000, [0]
    saw = {"dropped": 0, "low_put": 0, "rebuild": 0, "remote_unset": 0}

    def page():
        pid[0] += 1
        return datagen.make_page(KINDS[pid[0] % len(KINDS)], bs, 100_000 * seed + pid[0])

    def deliver(due):
        nonlocal pending
        for r in range(world):
            mine = [rows for (t, tgt, rows) in pending if tgt == r and t <= due]
            if not mine:
                continue
            rows = np.concatenate(mine)
            rows = rows[rng.permutation(len(rows))]
            d = engs[r].dev_alloc(rows.nbytes)
            engs[r].h2d(d, rows)
            engs[r].import_records_dev(len(rows), d, r)
            engs[r].sync()
            engs[r].dev_free(d)
            ua, la, sq, ow, ln = sharding.unpack_records(rows)
            models[r].import_rows([((int(np.uint64(ua[i])), int(np.uint64(la[i]))), int(sq[i]), int(ow[i]), ln[i] >= 0)
                                   for i in range(len(rows))])
        pending = [p for p in pending if p[0] > due]

    try:
        for step in range(12):
            gathered = []
            for r in range(world):
                n = int(rng.integers(8, 41))
                idx = rng.integers(0, len(pool), n)
                addr = [pool[int(i)] for i in idx]
                if n > 4:
                    addr[3] = addr[1]                                   # an in-batch duplicate
                valid = (rng.random(n) > 0.08).astype(np.uint8)
                pages = np.stack([page() for _ in range(n)])
                u, l = split(addr)
                engs[r].set_stream_order(pos + r, world)
                engs[r].wait(engs[r].put_step(u, l, pages, valid=valid, rank=r, records_dev=d_rec[r]))
                engs[r].sync()
                rec = np.zeros((n, 4), np.int64)
                engs[r].d2h(rec, d_rec[r])
                ln = sharding.unpack_records(rec)[4]
                saw["dropped"] += int(((ln < 0) & (valid == 1)).sum())
                models[r].put([(addr[i] if valid[i] else None, pos + r + world * i, ln[i] >= 0, pages[i])
                               for i in range(n)])
                used.update(a for a, v in zip(addr, valid) if v)
                gathered.append(rec)
            pos += world * 64
            rows = np.concatenate(gathered)
            for r in range(world):
                pending.append((step + int(rng.integers(0, 3)), r, rows))
            deliver(step)
            _model_check(E, engs, models, used, f"step {step}")
            if step % 3 != 2:
                continue
            deliver(10 ** 9)                                            # every row is in before the next ops
            _model_check(E, engs, models, used, f"flush {step}")
            r = int(rng.integers(0, world))
            eng, m = engs[r], models[r]
            # a put below an imported row of the same key: the row stays the winner
            rem = [a for a in m.remote_keys() if m.lookup(a)[0] == E.REMOTE]
            if rem:
                a = rem[int(rng.integers(0, len(rem)))]
                w_pos = m.winner[RM.fnv_key(*a)].pos
                eng.set_stream_order(w_pos - 1, world)
                pg = page()[None]
                eng.put(*split([a]), pg)
                m.put([(a, w_pos - 1, True, pg[0])])
                saw["low_put"] += 1
                _model_check(E, engs, models, used, f"low put {step}")
            # unsets of local and of remote keys
            loc = list(m.local_records())
            rem = m.remote_keys()
            pick = [loc[int(i)] for i in rng.permutation(len(loc))[:max(1, len(loc) // 4)]] + rem[:3]
            saw["remote_unset"] += len(rem[:3])
            eng.unset(*split(pick))
            m.unset(pick)
            _model_check(E, engs, models, used, f"unset {step}")
            eng.compact()
            _model_check(E, engs, models, used, f"compact {step}")
            if step == 5:
                # more than cap / 8 tombstones: 160 fresh local keys and every local key removed, then the
                # compaction rebuilds the table (on rank 0 or 1: rank 2's small arena drops most of them)
                r = r % 2
                eng, m = engs[r], models[r]
                cap = eng.stats()["table_slots"]
                extra = [(0xE000 + r, i) for i in range(160)]
                eng.set_stream_order(pos + r, world)
                pages = np.stack([page() for _ in extra])
                ln = eng.put(*split(extra), pages)
                m.put([(a, pos + r + world * i, ln[i] >= 0, pages[i]) for i, a in enumerate(extra)])
                used.update(extra)
                pos += world * len(extra)
                _model_check(E, engs, models, used, f"extra {step}")
                loc = list(m.local_records())
                eng.unset(*split(loc))
                m.unset(loc)
                assert eng.stats()["tombstones"] > cap // 8
                eng.compact()
                saw["rebuild"] += eng.stats()["tombstones"] == 0
                _model_check(E, engs, models, used, f"rebuild {step}")
            # save, then load into a fresh engine: the file holds exactly the local records
            path = str(tmp_path / f"r{r}s{step}.snap")
            assert eng.save(path) == m.entries()
            fresh = E.Engine(pshift=12, accel=12, table_slots=512, arena_bytes=32 << 20, max_batch=64, flags=E.VERIFY)
            try:
                assert fresh.load(path) == m.entries()
                _model_check(E, [fresh], [RM.ReplicaModel.loaded(0, m.local_records())], used, f"load {step}")
            finally:
                fresh.close()
            _, _, n_bad, checked = eng.verify_store()
            assert n_bad == 0 and checked == m.entries(), (n_bad, checked, m.entries())
        print(f"\n[replica model {seed}] {saw}")
        assert saw["dropped"] and saw["low_put"] and saw["remote_unset"] and saw["rebuild"]
    finally:
        for e, d in zip(engs, d_rec):
            e.dev_free(d)
            e.close()


# ---- a known limit of the replica (DESIGN.md §9): a tombstone keeps its position, not its key ---------

def _home_slot(key, cap):
    """kernels.cu home_slot: the key remixed, masked to the table."""
    z = ((key ^ (key >> 32)) * 0xD6E8FEB86659FD93) & 0xFFFFFFFFFFFFFFFF
    z ^= z >> 32
    return z & (cap - 1)


def _late_row_on_a_tombstone(E, row_pos):
    """Rank 1 puts address a at position 100 and unsets it: a's home slot becomes a tombstone that keeps
    position 100.  Then rank 0's row for address b, another key with the same home slot, is imported at
    `row_pos`; it claims that tombstone.  -> (status and owner of b on the engine, the model's answer)."""
    import replica_model as RM
    eng = E.Engine(pshift=12, accel=12, capacity=256, arena_bytes=8 << 20, max_batch=64)
    try:
        cap = eng.stats()["table_slots"]
        a = (0xF00D, 0)
        home = _home_slot(RM.fnv_key(*a), cap)
        b = next((0xF00D, i) for i in range(1, 1 << 20) if _home_slot(RM.fnv_key(0xF00D, i), cap) == home)
        m = RM.ReplicaModel(ME)
        page = datagen.make_page("T", 4096, 5)
        eng.set_stream_order(100, WORLD)
        assert eng.put(*split([a]), page[None])[0] > 0
        m.put([(a, 100, True, page)])
        eng.unset(*split([a]))
        m.unset([a])
        assert eng.stats()["tombstones"] == 1
        rows = sharding.pack_records([b[0]], [b[1]], [row_pos], 0, [200], [4096])
        d = eng.dev_alloc(rows.nbytes)
        eng.h2d(d, rows)
        eng.import_records_dev(len(rows), d, ME)
        eng.sync()
        eng.dev_free(d)
        m.import_rows([(b, row_pos, 0, True)])
        assert eng.stats()["tombstones"] == 0                   # b's claim took a's tombstone
        st, ow = eng.locate(*split([a, b]))
        assert st[0] == E.MISS
        return (int(st[1]), int(ow[1]) if st[1] == E.REMOTE else -1), m.lookup(b)[:2]
    finally:
        eng.close()


def test_a_row_above_the_tombstones_position_is_imported(E, gpu):
    got, want = _late_row_on_a_tombstone(E, 150)
    assert got == want == (E.REMOTE, 0)


@pytest.mark.xfail(strict=True, reason="DESIGN.md §9: a late row for a new key that claims a tombstone with a "
                                       "higher position is dropped (k_import_claim_rec atomicMax, then the seq check)")
def test_a_late_row_on_a_newer_tombstone_is_imported(E, gpu):
    got, want = _late_row_on_a_tombstone(E, 50)
    assert want == (E.REMOTE, 0)
    assert got == want                                            # today: (MISS, -1)
