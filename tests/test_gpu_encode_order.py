"""Longest-first handout of the encoder (DESIGN.md §4) through the store: batches with more chunks than
the encoder has resident warps on an H100 (132 SMs x 13 ring warps, x 14 plain warps), so that every
chunk is rated by k_cost and handed out from the cost buckets.  Whatever order the chunks are encoded
in, each must be encoded exactly once and land where its index says: stored lengths, records and
fingerprints equal the oracle's, and entries, dropped puts and garbage follow the store model."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
BS = 65536
N = 2304                   # > 132 x 14: the ordered handout runs in both encoder organisations


def class_cids(cls: int, n: int, first: int = 0) -> np.ndarray:
    """The first n chunk ids >= first of one class of the synthetic stream (R, T, Z, M = 0..3)."""
    c = np.arange(first, first + 8 * n, dtype=np.uint64)
    return c[((c + (c >> np.uint64(3))) & np.uint64(3)) == cls][:n]


def need(clen: int) -> int:
    return (24 + clen + 15) & ~15


def check_batch(E, oracle, eng, u, l, pages, lens, accel, valid=None):
    """lens == -1 exactly for the chunks a later chunk of the batch rewrites and for invalid addresses;
    every other chunk's record and fingerprint is the oracle's."""
    ok_addr = np.ones(len(u), dtype=bool) if valid is None else valid.astype(bool)
    last = {}
    for i, k in enumerate(zip(u.tolist(), l.tolist())):
        if ok_addr[i]:
            last[k] = i
    live = np.zeros(len(u), dtype=bool)
    live[list(last.values())] = True
    assert (lens[~live] == -1).all(), np.nonzero(lens[~live] != -1)
    idx = np.nonzero(live)[0]
    recs, rec_lens = eng.read_records_raw(u[idx], l[idx])
    par = oracle.parity_records(pages[idx], u[idx], l[idx], recs, rec_lens, lens[idx], accel)
    assert par["chunks"] == len(idx) and par["mismatches"] == 0, par
    fps, ok = eng.read_fingerprints(u[idx], l[idx])
    assert ok.all()
    for j, i in enumerate(idx):
        assert (int(fps[j, 0]), int(fps[j, 1])) == oracle.fingerprint128(pages[i]), i
    st = eng.stats()
    assert st["entries"] == len(idx) and st["dropped_puts"] == 0
    return st


@pytest.mark.parametrize("what", ["all_text", "costly_page_last"])
def test_ordered_handout_encodes_every_chunk_once(E, gpu, oracle, what):
    if what == "all_text":
        cids = class_cids(1, N)
    else:
        cids = np.append(class_cids(2, N - 1), class_cids(1, 1, first=8 * N))
    pages = oracle.gen_chunks(42, cids, BS)
    eng = E.Engine(pshift=16, accel=12, capacity=4 * N, arena_bytes=1 << 30, max_batch=4096, flags=E.FINGERPRINT)
    u = np.full(N, 5, dtype=np.uint64)
    l = np.arange(N, dtype=np.uint64)
    lens = eng.put(u, l, pages, on_dev=False)
    st = check_batch(E, oracle, eng, u, l, pages, lens, 12)
    assert st["arena_garbage"] >= 0
    out, status = eng.get(u[-4:], l[-4:])
    assert (status == E.HIT).all() and (out == pages[-4:]).all()
    eng.close()


@pytest.mark.parametrize("accel", [12, 17])       # 17: above the ring's limit, the plain organisation
def test_ordered_handout_with_duplicates_and_an_invalid_address(E, gpu, oracle, accel):
    cids = np.arange(N, dtype=np.uint64)
    pages = oracle.gen_chunks(7, cids, BS)
    u = np.full(N, 9, dtype=np.uint64)
    l = np.arange(N, dtype=np.uint64) % np.uint64(N - 300)      # the last 300 chunks rewrite earlier keys
    l[N - 40: N - 20] = l[N - 20:]                              # ... and some of them are rewritten again
    valid = np.ones(N, dtype=np.uint8)
    valid[[3, N // 2, N - 1]] = 0                               # invalid addresses: never stored, lens -1
    eng = E.Engine(pshift=16, accel=accel, capacity=4 * N, arena_bytes=1 << 30, max_batch=4096, flags=E.FINGERPRINT)
    lens = eng.put(u, l, pages, valid=valid)
    check_batch(E, oracle, eng, u, l, pages, lens, accel, valid)
    eng.close()


def test_ordered_handout_into_a_full_arena_reports_drops(E, gpu, oracle, monkeypatch):
    """Rewrite every key of a stored batch while the arena has room for about half of the new records:
    a put that does not fit is dropped and counted, its lens entry is -1 (it stored nothing), and its
    key still reads its old record."""
    monkeypatch.setenv("CMB200_SEG_KB", "0")                    # records through the stage: exact arena accounting
    a_cids = np.arange(N, dtype=np.uint64)
    b_cids = a_cids + np.uint64(4 * N)
    pa, pb = oracle.gen_chunks(3, a_cids, BS), oracle.gen_chunks(3, b_cids, BS)
    la = np.array([len(oracle.lz4_encode(p, 12)) for p in pa])
    lb = np.array([len(oracle.lz4_encode(p, 12)) for p in pb])
    na, nb = np.vectorize(need)(la), np.vectorize(need)(lb)
    arena = (int(na.sum()) + int(nb.sum()) // 2 + 255) & ~255
    eng = E.Engine(pshift=16, accel=12, capacity=4 * N, arena_bytes=arena, max_batch=4096, flags=E.FINGERPRINT)
    u = np.full(N, 13, dtype=np.uint64)
    l = np.arange(N, dtype=np.uint64)
    lens_a = eng.put(u, l, pa)
    check_batch(E, oracle, eng, u, l, pa, lens_a, 12)
    assert eng.stats()["arena_garbage"] == 0
    lens_b = eng.put(u, l, pb)
    out, status = eng.get(u, l)
    assert (status == E.HIT).all()
    new = np.array([(out[i] == pb[i]).all() for i in range(N)])
    old = np.array([(out[i] == pa[i]).all() for i in range(N)])
    assert (new ^ old).all(), "a key reads neither its old nor its new page"
    assert 0 < new.sum() < N
    # lens: the stored block's length, -1 exactly for the puts the full arena dropped
    assert (lens_b == np.where(new, lb, -1)).all()
    st = eng.stats()
    assert st["dropped_puts"] == int(old.sum())
    assert st["entries"] == N
    assert st["arena_garbage"] == int(na[new].sum())             # the records the stored puts replaced
    recs, rec_lens = eng.read_records_raw(u[new], l[new])
    par = oracle.parity_records(pb[new], u[new], l[new], recs, rec_lens, lens_b[new], 12)
    assert par["mismatches"] == 0, par
    eng.close()
