"""GPU: the LZ4 encoder on the encoder corpus (tests/lz4_encoder_corpus.py), whose pages reach every
branch the census (tests/test_lz4_encoder_census.py) counts, against the oracle.

Codec: each (page size, accel) group of the corpus through lz4_encode_batch with fingerprints, once
as a batch below the resident warp count (one page per warp, no k_cost) and once repeated to more
than 132 x 14 chunks (k_cost orders the batch; every warp encodes several pages in a row, reusing
its ring's mbarrier phases and clearing its table between pages).  Blocks equal oracle.lz4_encode
(and, on a seeded fifth of the pages, the reference's own LZ4_compress_fast where oracle/_ref was
built), fingerprints equal oracle.fingerprint128, and lz4_decode_batch gives the page back and
consumes the whole block.

Store: the corpus pages of one size through a store with FINGERPRINT, with records through the
stage rows (CMB200_SEG_KB=0) and straight into arena segments (the default): records, fingerprints
and the encoder's parse checkpoints against the oracle, pages through the batch get and (up to 2^17)
the fused get.

A block that differs is diffed sequence by sequence against the trace of the reference parse: the
message names the family, the page, the first differing sequence and its trace record.
"""
import collections

import numpy as np
import pytest

import datagen
import lz4_encoder_corpus as C
import lz4_trace as T
from ckpt_def import ckpt_words

pytestmark = pytest.mark.gpu
RESIDENT = 132 * 14                   # more chunks than an H100 has encoder warps: k_cost orders the batch
STORE_PSHIFTS = [6, 8, 10, 12, 16, 17, 18]
SMALL_GET_MAX = 17


@pytest.fixture(scope="module")
def corpus():
    return C.corpus()


def _seqs(block: bytes):
    """Token stream of a block: [(literal run, offset, match code, literal bytes)], the last literals as
    (run, None, None, literal bytes).  A malformed block ends the list where it runs out of bytes,
    with a None entry, so that a diagnosis never fails on the bytes it diagnoses."""
    out, ip, end = [], 0, len(block)

    def ext(v):
        nonlocal ip
        while ip < end:
            b = block[ip]
            ip += 1
            v += b
            if b != 255:
                return v
        return None

    while ip < end:
        tok = block[ip]
        ip += 1
        lit = tok >> 4 if tok >> 4 < 15 else ext(15)
        if lit is None:
            out.append(None)
            break
        lits = block[ip:ip + lit]
        ip += lit
        if ip >= end:
            out.append((lit, None, None, lits))
            break
        if ip + 2 > end:
            out.append(None)
            break
        off = block[ip] | block[ip + 1] << 8
        ip += 2
        mc = tok & 15 if tok & 15 < 15 else ext(15)
        if mc is None:
            out.append(None)
            break
        out.append((lit, off, mc, lits))
    return out


def diagnose(p, got: bytes, want: bytes) -> str:
    """Where two blocks of page p first differ, in the terms of the trace."""
    tr = T.parse(p.page, p.accel)
    steps = T.simulate(tr)
    a, b = _seqs(got), _seqs(want)
    i = next((j for j, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
    head = f"{p.family} {p.name} (n {p.n}, accel {p.accel}): {len(got)} vs {len(want)} bytes; first differing sequence #{i}"
    if i >= len(tr.seqs):
        return f"{head}: the last literals (run {tr.n - tr.last}, anchor {tr.last})"
    s, st = tr.seqs[i], steps[i]
    if i >= len(a) or a[i] is None:
        a = a[:i] + [("malformed", None, None, b"")]
    bins = []
    if s.lit <= 140:
        bins.append(f"B7 run {s.lit} x anchor&3 {s.anchor & 3}")
    if s.mc in C.MCS:
        bins.append(f"B8 match code {s.mc} after run {s.lit}")
    return (f"{head}: lane {s.lane} (probe {s.probe}, {'first search' if s.first else 'later search'}, "
            f"width {st.width}, path {st.path}), run {s.lit} at anchor {s.anchor} (anchor&3 {s.anchor & 3}), "
            f"match code {s.mc} (back {s.back}, fwd {s.fwd}), offset {s.off}; got {a[i][:3]}, want {b[i][:3]}"
            + ("" if a[i][3] == b[i][3] else f", literal bytes differ from offset "
               f"{next((j for j, (x, y) in enumerate(zip(a[i][3], b[i][3])) if x != y), '-')}")
            + (f"; {', '.join(bins)}" if bins else ""))


def _groups(corpus):
    g = collections.defaultdict(list)
    for p in corpus:
        g[p.n, p.accel].append(p)
    return sorted(g.items())


@pytest.mark.parametrize("repeat", ["one_page_per_warp", "ordered_many_per_warp"])
def test_codec_encodes_the_corpus(E, gpu, oracle, corpus, repeat):
    R = oracle.ref()
    for (n, accel), ps in _groups(corpus):
        want = [oracle.lz4_encode(p.page, accel) for p in ps]
        fp_want = [oracle.fingerprint128(p.page) for p in ps]
        reps = 1 if repeat == "one_page_per_warp" else RESIDENT // len(ps) + 1
        idx = np.tile(np.arange(len(ps)), reps)
        if repeat == "one_page_per_warp":
            assert len(ps) <= 132 * 13, (n, accel, len(ps))
        rows = datagen.pad_rows([ps[i].page for i in idx])
        blocks, fps = E.lz4_encode_batch(rows, nbytes=n, accel=accel, fingerprints=True)
        for j, i in enumerate(idx):
            assert blocks[j] == want[i], diagnose(ps[i], blocks[j], want[i])
            assert (int(fps[j, 0]), int(fps[j, 1])) == fp_want[i], (ps[i].name, j)
        if R is not None and repeat == "one_page_per_warp":
            pick = datagen.words(n * 31 + accel, len(ps)) % np.uint64(5) == 0
            for i in np.nonzero(pick)[0]:
                assert want[i] == oracle.ref_lz4_encode(ps[i].page, accel), ps[i].name
        out, used = E.lz4_decode_batch(blocks[:len(ps)], n)
        for i, p in enumerate(ps):
            assert used[i] == len(want[i]) and (out[i] == p.page).all(), (p.name, used[i], len(want[i]))


@pytest.mark.parametrize("records", ["stage_rows", "arena_segments"])
@pytest.mark.parametrize("pshift", STORE_PSHIFTS)
def test_store_encodes_the_corpus(E, gpu, oracle, corpus, monkeypatch, pshift, records):
    n = 1 << pshift
    ps = [p for p in corpus if p.n == n]
    assert ps, n
    if records == "stage_rows":
        monkeypatch.setenv("CMB200_SEG_KB", "0")
    k = len(ps)
    pages = np.stack([p.page for p in ps])
    u = np.full(k, 0xE7C0, dtype=np.uint64)
    l = np.arange(k, dtype=np.uint64)
    eng = E.Engine(pshift=pshift, accel=12, capacity=max(1024, 4 * k), arena_bytes=4 * k * (n + 2048) + (64 << 20),
                   max_batch=4096, flags=E.FINGERPRINT)
    try:
        lens = eng.put(u, l, pages)
        want = [oracle.lz4_encode(p.page, 12) for p in ps]
        recs, rec_lens = eng.read_records_raw(u, l)
        par = oracle.parity_records(pages, u, l, recs, rec_lens, lens, 12)
        if par["mismatches"]:
            i = par["first_mismatch"]
            got = recs[i, 24:24 + max(0, rec_lens[i] - 24)].tobytes()
            pytest.fail(f"{par}; " + diagnose(_at_store_accel(ps[i]), got, want[i]))
        fps, ok = eng.read_fingerprints(u, l)
        assert ok.all()
        for i, p in enumerate(ps):
            assert (int(fps[i, 0]), int(fps[i, 1])) == oracle.fingerprint128(p.page), p.name
        if pshift <= SMALL_GET_MAX:
            words, ok = eng.read_checkpoints(u, l)
            for i, p in enumerate(ps):
                if lens[i] > 0:
                    assert ok[i] == 1 and words[i, 1:].tolist() == ckpt_words(want[i], n)[1:], (p.name, ok[i])
        out, st = eng.get(u, l)
        assert (st == E.HIT).all() and (out == pages).all()
        if pshift <= SMALL_GET_MAX:
            for s in range(0, k, 512):
                out, st = eng.get_small(u[s:s + 512], l[s:s + 512])
                assert (st == E.HIT).all() and (out == pages[s:s + 512]).all(), s
        assert eng.stats()["dropped_puts"] == 0
    finally:
        eng.close()


def _at_store_accel(p):
    """The page as the store encodes it: at the store's acceleration, 12."""
    return C.Page(p.family, p.name, 12, p.page)
