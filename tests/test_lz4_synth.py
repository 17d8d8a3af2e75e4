"""CPU: the synthesized LZ4 blocks (tests/lz4_synth.py) against the oracle and the reference's
decoder, and the limited-output rule of filemap_set (LZ4_compress_fast into bsize + 1024 bytes)
against the reference's return values (tests/golden/lz4_limit.json)."""
import json
import os

import pytest

import ckpt_def
import datagen
import lz4_synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SIZES = [1 << p for p in range(6, 21)]


@pytest.mark.parametrize("n", SIZES)
def test_synthesized_blocks_decode_to_their_pages(oracle, n):
    R = oracle.ref()
    cases = lz4_synth.cases(n)
    families = {c.family for c in cases}
    assert {"F1", "F2", "F3", "F4", "F5", "F6", "F8"} <= families, families
    if n >= 1 << 17:
        assert "F7" in families
    for c in cases:
        page, used = oracle.lz4_decode(c.block, n)
        if not c.valid:
            assert used != len(c.block), c.name            # every twin breaks a rule the oracle checks
            continue
        assert len(c.page) == n
        assert used == len(c.block) and page == c.page, (c.name, used, len(c.block))
        assert ckpt_def.ckpt_words(c.block, n) is not None, c.name
        if R is not None:                                   # trusting decoder: valid blocks only
            rpage, rused = oracle.ref_lz4_decode(c.block, n)
            assert rused == len(c.block) and rpage == c.page, (c.name, rused)


def test_synthesized_blocks_reach_the_edges():
    """The shapes the families promise are in the blocks, parsed back from the bytes."""
    def seqs(block):
        ip, op, out = 0, 0, []
        while True:
            tok = block[ip]; ip += 1
            lit = tok >> 4
            if lit == 15:
                while True:
                    b = block[ip]; ip += 1; lit += b
                    if b != 255:
                        break
            ip += lit; op += lit
            if ip == len(block):
                return out, op, lit
            off = block[ip] | block[ip + 1] << 8; ip += 2
            ml = tok & 15
            if ml == 15:
                while True:
                    b = block[ip]; ip += 1; ml += b
                    if b != 255:
                        break
            out.append((op - lit, lit, op, off, ml + 4))
            op += ml + 4

    n = 1 << 17
    got = {"off": set(), "to": set(), "lit": set(), "lit_at": set(), "mlen": set()}
    ends = set()
    for c in lz4_synth.cases(n):
        if not c.valid:
            continue
        ss, _, last = seqs(c.block)
        for lit_at, lit, to, off, mlen in ss:
            got["off"].add(off); got["to"].add((off, to & 15)); got["mlen"].add(mlen)
            got["lit"].add(lit); got["lit_at"].add((lit, lit_at & 15))
            if to == off:
                ends.add("off_eq_op")
            if to + mlen == n - 5:
                ends.add("match_to_n-5")
            if lit_at + lit == n - 9 and mlen == 4:
                ends.add("lits_to_n-9")
        if last == 5:
            ends.add("last_run_5")
    assert set(lz4_synth.OFFSETS) <= got["off"]
    assert all((off, a) in got["to"] for off in range(1, 141) for a in range(16))
    assert set(lz4_synth.LENGTHS) <= got["mlen"] and {f + 4 for f in lz4_synth.FIELDS} <= got["mlen"]
    assert set(lz4_synth.FIELDS) <= got["lit"] and any(x >= 65536 for x in got["lit"])
    assert all((L, a) in got["lit_at"] for L in range(71) for a in range(16))
    assert any(m - 4 >= 65536 for m in got["mlen"])
    assert ends == {"off_eq_op", "match_to_n-5", "lits_to_n-9", "last_run_5"}


def _limit_cases():
    return json.load(open(os.path.join(GOLD, "lz4_limit.json")))["cases"]


def test_limited_output_rule_matches_the_reference(oracle):
    """filemap_set calls LZ4_compress_fast(page, dst, n, n + 1024): the reference refuses a page
    (returns 0) exactly when the unlimited block is longer than n + 1024, else returns that block."""
    cases = _limit_cases()
    assert {r[0] for r in cases} == {17, 18, 19, 20}
    refused = [r for r in cases if r[5] == 0]
    assert refused and len(refused) < len(cases)
    R = oracle.ref()
    for pshift, accel, seed, at, z, ref_len in cases:
        n = 1 << pshift
        page = datagen.limit_page(n, seed, at, z)
        blk = oracle.lz4_encode(page, accel)
        assert (len(blk) > n + 1024) == (ref_len == 0), (pshift, accel, seed, z, len(blk))
        if ref_len:
            assert len(blk) == ref_len
        if R is not None:
            assert len(oracle.ref_lz4_encode(page, accel)) == ref_len


def test_store_model_keeps_refused_pages_raw(oracle):
    """The store keeps a page the reference refuses as a raw record (compressed_length 0)."""
    for i, (pshift, accel, seed, at, z, ref_len) in enumerate(_limit_cases()):
        n = 1 << pshift
        page = datagen.limit_page(n, seed, at, z)
        model = oracle.StoreModel(pshift, accel)
        off, nh = (i + 1) << pshift, 0x5EED
        model.put(off, nh, 0, page)
        u, l = oracle.addr_compose(off, nh, 0, pshift)
        rec = model.record_bytes(u, l)
        clen = int.from_bytes(rec[16:20], "little")
        if ref_len == 0:
            assert clen == 0 and rec[24:] == page.tobytes(), (pshift, seed, z)
        else:
            assert clen == ref_len and len(rec) == 24 + ref_len
        assert len(rec) <= 24 + n + 1024
        assert model.get(off, nh, 0) == page.tobytes()
