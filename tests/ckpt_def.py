"""Independent Python statement of the parse checkpoints (edge_fuse_b200/csrc/kernels.h) that the
encoder leaves per record and k_restore rebuilds from a loaded block.  Test helper, CPU only."""
from __future__ import annotations

CKPT_WORDS, CKPT_POS_BITS = 16, 13
NONE = 0xFFFFFFFF


def ckpt_words(block, n: int):
    """Parse checkpoints of an LZ4 block of a page of n bytes: a list of 16 ints (word 0, the tag, is
    0 here), or None when the token chain does not end exactly at (len(block), n).  Every token starts
    a sequence, the last literal-only one included; with S = n // 16, word k (1..15) is set by the
    first sequence whose literals start at lit_start >= k * S: ip << 13 | (lit_start - k * S) when
    that distance is below S, else ~0 (also when no such sequence exists)."""
    blk = bytes(block)
    S = n // CKPT_WORDS
    seqs = []                                       # (token offset, output position of its literals)
    ip = op = 0
    while True:
        if ip >= len(blk):
            return None
        seqs.append((ip, op))
        tok = blk[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if ip >= len(blk):
                    return None
                b = blk[ip]
                ip += 1
                lit += b
                if b != 255:
                    break
        if lit > n - op or ip + lit > len(blk):
            return None
        ip += lit
        op += lit
        if ip == len(blk):
            break
        if ip + 2 > len(blk):
            return None
        ip += 2
        mlen = tok & 15
        if mlen == 15:
            while True:
                if ip >= len(blk):
                    return None
                b = blk[ip]
                ip += 1
                mlen += b
                if b != 255:
                    break
        if op + mlen + 4 > n:
            return None
        op += mlen + 4
    if op != n:
        return None
    words = [0] + [NONE] * (CKPT_WORDS - 1)
    for k in range(1, CKPT_WORDS):
        first = next(((sip, sop) for sip, sop in seqs if sop >= k * S), None)
        if first is not None and first[1] - k * S < S:
            words[k] = (first[0] << CKPT_POS_BITS) | (first[1] - k * S)
    return words
