"""The parse-checkpoint definition restated in ckpt_def.ckpt_words (kernels.h, lz4_encode_lean): known
answers worked by hand, the rule that the sections the words name add up to the serial parse of the
reference's own blocks (tests/golden/lz4_blocks.json), and None for chains that do not fit.  CPU only."""
import hashlib
import json
import os

import numpy as np

import datagen
from ckpt_def import NONE, ckpt_words

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _len_bytes(v):
    """LZ4 length extension bytes for a length field value v >= 15 (the nibble holds 15)."""
    v -= 15
    return [255] * (v // 255) + [v % 255]


def _block(seqs, last_lits):
    """An LZ4 block from (literal bytes, offset, match length) sequences and the last literals."""
    out = bytearray()
    for lits, off, mlen in list(seqs) + [(last_lits, 0, 0)]:
        last = off == 0
        m = mlen - 4
        out.append((min(len(lits), 15) << 4) | (0 if last else min(m, 15)))
        if len(lits) >= 15:
            out += bytes(_len_bytes(len(lits)))
        out += bytes(lits)
        if last:
            break
        out += off.to_bytes(2, "little")
        if m >= 15:
            out += bytes(_len_bytes(m))
    return bytes(out)


def _walk(blk, ip, op, op_end, n):
    """Sequences from (ip, op) while op < op_end, as dc_parse_chain takes a section -> (ip, op)."""
    while op < op_end:
        tok = blk[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = blk[ip]
                ip += 1
                lit += b
                if b != 255:
                    break
        ip += lit
        op += lit
        if op == n:
            break
        ip += 2
        m = tok & 15
        if m == 15:
            while True:
                b = blk[ip]
                ip += 1
                m += b
                if b != 255:
                    break
        op += m + 4
    return ip, op


def _sections_fit(words, blk, n):
    """The rule of gs_sections_fit: the section from each named (ip, op) ends where the next named one
    starts, the last at (len(blk), n)."""
    S = n // 16
    starts = [(0, 0)]
    for k in range(1, 16):
        if words[k] == NONE:
            continue
        ip, rel = words[k] >> 13, words[k] & 0x1FFF
        assert rel < S and ip < len(blk) and ip > starts[-1][0]
        starts.append((ip, k * S + rel))
    for (ip, op), nxt in zip(starts, starts[1:] + [None]):
        end = _walk(blk, ip, op, nxt[1] if nxt else n, n)
        if end != (nxt if nxt else (len(blk), n)):
            return False
    return True


def test_zero_page_is_one_match_and_the_last_literals(oracle):
    for n in (4096, 65536, 131072):
        blk = oracle.lz4_encode(np.zeros(n, dtype=np.uint8), 12)
        w = ckpt_words(blk, n)
        S = n // 16
        # the last literals are the 5 bytes LZ4 keeps after the last match: token + 5 literals end the block
        assert w[1:15] == [NONE] * 14
        assert w[15] == ((len(blk) - 6) << 13) | (n - 5 - 15 * S)
        assert _sections_fit(w, blk, n)


def test_single_literal_sequence(oracle):
    n = 4096
    page = datagen.make_page("R", n, 3)
    blk = _block([], page.tobytes())
    assert blk[:18] == bytes([0xF0] + [255] * 16 + [1]) and len(blk) == 18 + n
    assert oracle.lz4_decode(blk, n) == (page.tobytes(), len(blk))
    assert ckpt_words(blk, n) == [0] + [NONE] * 15


def test_empty_sections_and_a_sequence_on_a_boundary(oracle):
    n, S = 4096, 256
    lits = datagen.make_page("R", 310, 9).tobytes()
    # A: 300 literals at 0, match to 512 = 2 S;  B: 10 literals at 512, match to n - 5;  last 5 literals
    blk = _block([(lits[:300], 1, 212), (lits[300:310], 7, n - 5 - 522)], b"\x01\x02\x03\x04\x05")
    page, used = oracle.lz4_decode(blk, n)
    assert used == len(blk) == 339
    w = ckpt_words(blk, n)
    want = [0] + [NONE] * 15
    want[2] = 306 << 13 | 0                           # B's token at 306, its literals exactly at 2 S
    want[15] = 333 << 13 | (n - 5 - 15 * S)           # the last literals at 4091
    assert w == want                                  # sections 1 and 3..14 are empty
    assert _sections_fit(w, blk, n)


def test_golden_blocks_sections_fit(oracle):
    with open(os.path.join(GOLD, "lz4_blocks.json")) as f:
        cases = json.load(f)["cases"]
    seen = 0
    for rec in cases:
        n = rec["n"]
        if n < 4096 or n > 131072 or n & (n - 1):
            continue
        page = datagen.make_page(rec["kind"], n, rec["seed"])
        blk = oracle.lz4_encode(page, rec["accel"])
        assert hashlib.sha256(blk).hexdigest() == rec["sha256"], rec
        w = ckpt_words(blk, n)
        assert w is not None and w[0] == 0, rec
        assert _sections_fit(w, blk, n), rec
        seen += 1
    assert seen >= 40


def test_chains_that_do_not_fit(oracle):
    n = 16384
    page = datagen.make_page("T", n, 21)
    blk = oracle.lz4_encode(page, 12)
    assert ckpt_words(blk, n) is not None
    assert ckpt_words(blk[:-1], n) is None                  # truncated last literals
    assert ckpt_words(blk[:len(blk) // 2], n) is None       # cut inside the chain
    assert ckpt_words(blk + b"\x00", n) is None             # a byte past the last literals
    assert ckpt_words(blk, n - 16) is None                  # decodes to more than the page
    assert ckpt_words(blk, n + 16) is None                  # to less
    bad = bytearray(blk)
    bad[0] = 0xFF                                           # literal run past the block end
    assert ckpt_words(bytes(bad), n) is None
    assert ckpt_words(b"", n) is None
