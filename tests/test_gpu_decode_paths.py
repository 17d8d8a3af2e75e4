"""GPU: every LZ4 decoder on blocks that this project's encoder does not write, against the oracle.

The blocks come from tests/lz4_synth.py (families F1-F8, every page size 2^6-2^20).  They reach the
decoders through the codec call (k_decode, `lz4_decode_warp`) and through a store loaded from a
snapshot, read by the batch get (k_decode) and by the fused get (k_get_small, `lz4_decode_cta.cuh`,
and its two-CTA PAIR variant at 2^17), with parse checkpoints, without them (CMB200_CKPT=0), and
with half of the records demoted to the host tier (the fused get's non-TMA record staging).
Valid blocks must give the intended page and consume the whole block; every F8 twin must give
consumed != len / BAD_DECODE, never a HIT.

Decoder branch                                                     family that reaches it
`dc_match_wide`: off >= 136 and len >= 64 (128-byte steps, to & 3)    F1 (off 136-140, 255, 256, 4095,
                                                                    4096, 65535; every to & 15), F7
`dc_match_wide`: 32 <= off < 136                                    F1, F7 (off 32, 135)
`dc_match_wide`: off < 32, len < 4096                               F1 (off 1-31 x lengths to 271), F3
`dc_match_wide`: off < 32, len >= 4096 (16-byte periodic fill,      F1 (off 1-31 x 4096, 4097, 8175,
  period / first per off)                                           8200), F2 (match fields 8175+), F7
`dc_matches`: narrow overlapping / non-overlapping waves            F1 (off < len / off >= len), F3, F4
`dc_literals` wave analysis: chains up to 31 deep in a batch of    F3 (depth 2-40, skewed by 0-33
  32, and across batch and section edges                            independent sequences; F3.edges)
PAIR 17-bit fields: match length - 4 >= 65 536, literal length     F7 (2^17 and up)
  >= 65 536 (bit 31 of the literal word), destinations > 65 536
lane-copied literal runs (<= 64, every alignment); warp-copied      F4 (0-70 at every to & 15; 100,
  runs (> 64)                                                       1000, 5000), F2
length fields of exactly 270 (255, 0: `flen/fm == 270` of the      F2 (fields 269, 270, 525)
  fast parse)
runs of more than 32 0xFF bytes (`dcs_ext` / `lz4_read_ext` loops)  F2 (8430, 12000), F7
checkpoints at k n/16 and k n/16 + n/16 - 1 (8191 at 2^17, the      F6 (start, end, sparse)
  largest 13-bit value), empty sixteenths
block end: match to n - 5, literals to n - 9, final run of 5,       F5
  offset == op
rejected: match to n - 4, literals to n - 8 .. n - 1 before a       F8
  match, offset op + 1, offset 0, trailing byte, truncated
  extensions
"""
import numpy as np
import pytest

import lz4_synth
from ckpt_def import ckpt_words

pytestmark = pytest.mark.gpu
PSHIFTS = list(range(6, 21))
SMALL_GET_MAX = 17                    # the fused get serves pages up to 2^17


@pytest.mark.parametrize("pshift", PSHIFTS)
def test_codec_decoder(E, gpu, pshift):
    n = 1 << pshift
    cases = lz4_synth.cases(n)
    out, used = E.lz4_decode_batch([c.block for c in cases], n)
    for i, c in enumerate(cases):
        if c.valid:
            assert used[i] == len(c.block) and out[i].tobytes() == c.page, (c.name, used[i], len(c.block))
        else:
            assert used[i] != len(c.block), c.name


def _expect(E, cases, out, st, what):
    for i, c in enumerate(cases):
        if c.valid:
            assert st[i] == E.HIT and out[i].tobytes() == c.page, (what, c.name, st[i])
        else:
            assert st[i] == E.BAD_DECODE, (what, c.name, st[i])


def _get_small(eng, u, l, step=512):
    outs, sts = zip(*(eng.get_small(u[i:i + step], l[i:i + step]) for i in range(0, len(u), step)))
    return np.concatenate(outs), np.concatenate(sts)


@pytest.mark.parametrize("mode", ["ckpt", "no_ckpt", "host_tier"])
@pytest.mark.parametrize("pshift", PSHIFTS)
def test_store_decoders(E, gpu, oracle, tmp_path, monkeypatch, pshift, mode):
    from oracle import snapshot
    n = 1 << pshift
    cases = lz4_synth.cases(n)
    k = len(cases)
    assert all(len(c.block) <= n + 1024 for c in cases)     # what a snapshot may hold (filemap.c:120)
    u = np.full(k, 0x5157, dtype=np.uint64)
    l = np.arange(k, dtype=np.uint64)
    recs = [(i + 1, 0, 0, oracle.record_prefix(int(u[i]), int(l[i]), len(c.block)) + c.block) for i, c in enumerate(cases)]
    path = str(tmp_path / "synth.snap")
    snapshot.write_snapshot(path, pshift, recs)
    if mode == "no_ckpt":
        monkeypatch.setenv("CMB200_CKPT", "0")
    total = sum((len(r[3]) + 15) // 16 * 16 for r in recs)
    eng = E.Engine(pshift=pshift, accel=12, capacity=max(1024, 2 * k), arena_bytes=2 * total + (64 << 20),
                   max_batch=256, host_tier_bytes=2 * total + (64 << 20) if mode == "host_tier" else 0)
    try:
        assert eng.load(path) == k
        if mode == "host_tier":
            assert eng.demote(u[::2], l[::2]) == len(u[::2])
        out, st = eng.get(u, l)
        _expect(E, cases, out, st, "get")
        if pshift <= SMALL_GET_MAX:
            out, st = _get_small(eng, u, l)
            _expect(E, cases, out, st, "get_small")
            words, ok = eng.read_checkpoints(u, l)
            for i, c in enumerate(cases):
                if mode == "no_ckpt":
                    assert ok[i] == -1, c.name
                elif c.valid:
                    assert ok[i] == 1 and words[i, 1:].tolist() == ckpt_words(c.block, n)[1:], (c.name, ok[i])
        assert eng.stats()["dropped_puts"] == 0
    finally:
        eng.close()
