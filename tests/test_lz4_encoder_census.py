"""CPU: which branches of the warp LZ4 encoder the encoder corpus (tests/lz4_encoder_corpus.py) reaches,
counted by the traced reference parse (tests/lz4_trace.py), and the trace pinned to the oracle.

A cell counts what the trace saw on the corpus, never what a family planned.  Cells per bin (the
GPU side is tests/test_gpu_encode_paths.py):

  B1 winner lane      lane 1 (re-test), each probe lane 2-31, none within the batch; first search of a
                      page and later searches; x accel 1, 4, 12, 13, 17
  B2 narrow batch     16-lane batch whose winner is at lane 12-15 (widens again), at 16-31 (lz4_search_slow
                      from slot 16), beyond lane 31; a 16-lane batch with lanes cut by the end margin
  B3 aliases          two enabled lanes on one slot, the later at or below the winner: lane 0 + lane 1,
                      lane 0 or 1 + a probe lane, two probe lanes; byU16 and byU32
  B4 long searches    hit at probe 30-63, 64, 65, 127-129, >= 192; accel 1 and 12
  B5 forward ext.     3-35 bytes past hit + 4; lz4_count_long's step stage by 16-byte lane of its first
                      512-byte step and of a later one, and by pa & 3 x pb & 3; capped by mlimit in the
                      byte stage and in the step stage (the stage from the path's origin: hit + 8 in
                      the fast path, hit + 4 behind lz4_search_slow)
  B6 backward ext.    0-3, 4, 5-35, >= 36; stopped by the anchor; stopped by position 0; the fast path's
                      guards at back = 4: hit = anchor + 4, candidate = 4
  B7 literal runs     every run 0-140 x anchor & 3; 255-258, 269-271, >= 1000; runs 120-128 whose
                      speculative words cross the wrap of the 1 KiB ring
  B8 match codes      14-16, 268-271, 524, 525 after a run <= 128 and after a run of 129
  B9 ring            a sequence that jumps 256, 512, 768, 1024, >= 1280 bytes and ends at mod 256 in 0-7,
                      252-255; anchors at 256 g + 3, 4, 5; ragged last buffers (sizes not a multiple of 16)
  B10 block end       last match ending at mflimit - 1, mflimit, mflimit + 1, mlimit; a search that runs
                      into the margin inside the batch and inside lz4_search_slow; every size 13-40
  B11 far offsets     byU32: a candidate at 65 535 (taken), 65 536 and 65 537 (passed over), met by the
                      re-test, a batch lane (probes 0-29) and lz4_search_slow (probes from 30)
  B12 checkpoints     store sizes 2^6-2^17: sequences starting at k n/16 and k n/16 - 1, matches that
                      cover two or more sixteenth boundaries

Impossible cells are dropped by name in IMPOSSIBLE, with the reason.
"""
import collections
import json
import os
import time

import pytest

import datagen
import lz4_encoder_corpus as C
import lz4_trace as T

GOLD = os.path.join(os.path.dirname(__file__), "golden")

# Cells no page can reach.  A match starts at position 1 at the earliest and is at least 4 bytes long,
# so it ends at 5 or later; and a page of 13 bytes has mflimit 1, so its first probe (which needs the
# next probe position 2 <= mflimit) is never made.
_ENDS = (("mflimit-1", 13), ("mflimit", 12), ("mflimit+1", 11), ("mlimit", 5))
IMPOSSIBLE = {("B10", "end", d, n): "no match can end there" for d, back in _ENDS for n in range(13, 41)
              if n == 13 or n - back < 5}
# At 65 547 bytes mflimit is 65 535: a probe lies below it, so no probe meets a candidate 65 535 bytes
# back, and nothing at all lies 65 536 or more bytes past position 0 up to mflimit.
IMPOSSIBLE.update({("B11", 65547, d, f): "no position that far from 0 is searched"
                   for d in ("65535 taken", "65536 passed", "65537 passed") for f in ("retest", "lane", "slow")
                   if (d, f) != ("65535 taken", "retest")})


@pytest.fixture(scope="module")
def traced():
    t0 = time.time()
    pages = C.corpus()
    out = []
    for p in pages:
        tr = T.parse(p.page, p.accel)
        out.append((p, tr, T.simulate(tr)))
    return out, time.time() - t0


def census(traced):
    c = collections.Counter()
    amb = collections.Counter()
    for p, tr, steps in traced:
        a = p.accel
        for s, st in zip(tr.seqs, steps):
            when = "first" if s.first else "later"
            c["B1", a, when, s.lane if s.lane >= 0 else "none"] += 1
            if st.path == "ambiguous":
                amb["straddle", "byU32" if tr.wide else "byU16"] += 1
            if st.path == "unknown":
                amb["unknown width"] += 1
            if st.width == T.NARROW_W:
                if st.path == "fast" and s.lane >= 12:
                    c["B2", "widen 12-15"] += 1
                elif st.path == "slow_w" and 16 <= s.lane:
                    c["B2", "slow from 16"] += 1
                elif st.path == "slow_w" and s.lane < 0:
                    c["B2", "beyond 31"] += 1
                if st.narrow_cut:
                    c["B2", "cut by the margin"] += 1
            if st.path == "slow0":
                win = s.lane if s.lane >= 0 else T.LANES
                for g in T._alias_groups(s.en & ((1 << (st.width or T.LANES)) - 1), s.slots):
                    if g[1] <= win:
                        kind = "lane 0 + lane 1" if g[:2] == [0, 1] else "special + probe" if g[0] < 2 else "probe + probe"
                        c["B3", kind, "byU32" if tr.wide else "byU16"] += 1
            if a in (1, 12) and s.probe >= 30:
                k = s.probe
                cls = "30-63" if k < 64 else "64" if k == 64 else "65" if k == 65 else \
                    "127-129" if 127 <= k <= 129 else ">=192" if k >= 192 else None
                if cls:
                    c["B4", a, cls] += 1
            if 3 <= s.fwd <= 35:
                c["B5", "fwd", s.fwd] += 1
            fast, slow = st.path == "fast", st.path in ("slow0", "slow_w")
            if fast or slow:
                r = s.fwd - 4 if fast else s.fwd           # what lz4_count_long returns on this path
                capped = s.end == tr.mlimit
                if r >= 32:
                    q = r - 32
                    c["B5", "step1" if q < 512 else "step2+", (q % 512) // 16] += 1
                    c["B5", "pa&3 pb&3", s.hit & 3, s.cand & 3] += 1
                    if capped:
                        c["B5", "mlimit cap", "step stage"] += 1
                elif r >= 0 and capped:
                    c["B5", "mlimit cap", "byte stage"] += 1
            if fast and s.back == 4 and s.hit == s.anchor + 4:
                c["B6", "guard: hit = anchor + 4"] += 1
            if fast and s.back == 4 and s.cand == 4:
                c["B6", "guard: candidate = 4"] += 1
            b = s.back
            c["B6", "0-3" if b < 4 else "4" if b == 4 else "5-35" if b <= 35 else ">=36"] += 1
            if b and s.ip == s.anchor:
                c["B6", "stopped by the anchor"] += 1
            if b and s.cand - b == 0:
                c["B6", "stopped by position 0"] += 1
            if s.lit <= 140:
                c["B7", s.lit, s.anchor & 3] += 1
            for lo, hi in ((255, 258), (269, 271)):
                if lo <= s.lit <= hi:
                    c["B7", s.lit] += 1
            if s.lit >= 1000:
                c["B7", ">=1000"] += 1
            ring = a <= C.RING_MAX_ACCEL
            if ring and 120 <= s.lit <= 128 and s.anchor % 1024 > 1024 - s.lit:
                c["B7", "ring wrap", s.lit] += 1
            jump = s.end - s.anchor
            if ring and jump >= 256 and (s.end % 256 < 8 or s.end % 256 >= 252):
                c["B9", "jump", min(jump // 256, 5) * 256, s.end % 256] += 1
            if ring and s.anchor >= 256 and s.anchor % 256 in (3, 4, 5):
                c["B9", "anchor 256g+", s.anchor % 256] += 1
            if tr.wide:
                if s.off == 65535:
                    c["B11", tr.n, "65535 taken", C.far_finder(s.probe)] += 1
                for k, d in s.far:
                    if d in (65536, 65537):
                        c["B11", tr.n, f"{d} passed", C.far_finder(k)] += 1
            if tr.n in C.STORE_SIZES[:-1]:
                S = tr.n // 16
                if s.anchor % S == 0 and 0 < s.anchor < 16 * S:
                    c["B12", tr.n, "start k n/16"] += 1
                if (s.anchor + 1) % S == 0 and 0 < s.anchor + 1 < 16 * S:
                    c["B12", tr.n, "start k n/16 - 1"] += 1
                if s.end // S - s.ip // S >= 2:
                    c["B12", tr.n, "match over sixteenths"] += 1
            if s.mc in C.MCS and (s.lit <= 128 or s.lit == 129):
                c["B8", s.mc, "run<=128" if s.lit <= 128 else "run 129"] += 1
        if tr.n % 16 and p.accel <= C.RING_MAX_ACCEL:
            c["B9", "ragged", tr.n] += 1
        if tr.n >= T.MIN_INPUT:
            c["B10", "size", tr.n] += 1 if tr.n <= 40 else 0
            if tr.seqs:
                e = tr.seqs[-1].end
                for name, v in (("mflimit-1", tr.mflimit - 1), ("mflimit", tr.mflimit),
                                ("mflimit+1", tr.mflimit + 1), ("mlimit", tr.mlimit)):
                    if e == v:
                        c["B10", "end", name, tr.n] += 1
            if tr.tail_batch is not None:
                c["B10", "margin in the batch" if tr.tail_probes < 30 else "margin in lz4_search_slow"] += 1
    return c, amb


def minimums():
    m = {}
    for a in C.ACCELS:
        for lane in list(range(2, 32)) + ["none"]:
            m["B1", a, "first", lane] = 5
        for lane in list(range(1, 32)) + ["none"]:
            m["B1", a, "later", lane] = 5
    for k in ("widen 12-15", "slow from 16", "beyond 31", "cut by the margin"):
        m["B2", k] = 10
    for w in ("byU16", "byU32"):
        for kind in ("lane 0 + lane 1", "special + probe", "probe + probe"):
            m["B3", kind, w] = 5
    for a in (1, 12):
        for k in ("30-63", "64", "65", "127-129", ">=192"):
            m["B4", a, k] = 3
    for f in range(3, 36):
        m["B5", "fwd", f] = 2
    for st in ("step1", "step2+"):
        for lane in range(32):
            m["B5", st, lane] = 2
    for a3 in range(4):
        for b3 in range(4):
            m["B5", "pa&3 pb&3", a3, b3] = 2
    for st in ("byte stage", "step stage"):
        m["B5", "mlimit cap", st] = 2
    for k in ("0-3", "4", "5-35", ">=36", "stopped by the anchor", "stopped by position 0",
              "guard: hit = anchor + 4", "guard: candidate = 4"):
        m["B6", k] = 3
    for L in range(141):
        for a in range(4):
            m["B7", L, a] = 2
    for L in (255, 256, 257, 258, 269, 270, 271, ">=1000"):
        m["B7", L] = 2
    for L in range(120, 129):
        m["B7", "ring wrap", L] = 2
    for mc in C.MCS:
        for r in ("run<=128", "run 129"):
            m["B8", mc, r] = 3
    for J in (256, 512, 768, 1024, 1280):
        for t in list(range(8)) + list(range(252, 256)):
            m["B9", "jump", J, t] = 3
    for t in (3, 4, 5):
        m["B9", "anchor 256g+", t] = 3
    for n in C.CODEC_SIZES:
        if n % 16:
            m["B9", "ragged", n] = 3
    for n in (65547, 1 << 17, 1 << 18):
        for d in ("65535 taken", "65536 passed", "65537 passed"):
            for f in ("retest", "lane", "slow"):
                m["B11", n, d, f] = 3
    for n in C.STORE_SIZES[:-1]:
        for k in ("start k n/16", "start k n/16 - 1", "match over sixteenths"):
            m["B12", n, k] = 3
    for n in range(13, 41):
        m["B10", "size", n] = 1
    for n in C.CODEC_SIZES:
        for d in ("mflimit-1", "mflimit", "mflimit+1", "mlimit"):
            m["B10", "end", d, n] = 1
    for k in ("margin in the batch", "margin in lz4_search_slow"):
        m["B10", k] = 3
    return {k: v for k, v in m.items() if k not in IMPOSSIBLE}


def test_trace_rebuilds_the_oracle_blocks(oracle, traced):
    rows, _ = traced
    bad = [p.name for p, tr, _ in rows if tr.block() != oracle.lz4_encode(p.page, p.accel)]
    assert not bad, bad[:10]


def test_trace_rebuilds_the_golden_blocks(oracle):
    g = json.load(open(os.path.join(GOLD, "lz4_blocks.json")))["cases"]
    for r in g:
        if r["kind"] == "S":
            page = oracle.gen_chunks(42, [r["seed"]], r["n"])[0]
        else:
            page = datagen.make_page(r["kind"], r["n"], r["seed"])
        blk = T.parse(page, r["accel"]).block()
        assert len(blk) == r["len"] and blk == oracle.lz4_encode(page, r["accel"]), (r["kind"], r["n"], r["accel"])


def test_every_cell_is_reached(traced):
    rows, seconds = traced
    c, amb = census(rows)
    mins = minimums()
    short = {k: (c[k], v) for k, v in mins.items() if c[k] < v}
    lines = [f"{'/'.join(map(str, k)):40s} {c[k]:7d} >= {v}" for k, v in sorted(mins.items(), key=str)]
    print("\n".join(lines))
    print("ambiguous aliases (reported, not required):", dict(amb))
    print(f"corpus: {len(rows)} pages, {sum(len(t.seqs) for _, t, _ in rows)} sequences, {seconds:.1f} s")
    assert not short, "cells below their minimum (count, minimum): " + ", ".join(
        f"{'/'.join(map(str, k))}: {v}" for k, v in sorted(short.items(), key=str))
    assert seconds < 60, seconds
