"""Store addresses with a chosen 64-bit FNV-1a key, found with a small lattice reduction.

The store keys a 16-byte address {u, l} (u first, both little-endian) by FNV-1a-64 of its bytes.  Write
each step as h' = (h + d) * P with d = (h ^ b) - h: the final hash is a linear form in the d's,

    h_16 = h_k * P^(16-k) + sum_{i>k} d_i * P^(16-i+1)   (mod 2^64)

for any fixed prefix of k bytes.  A short vector of an integer lattice gives small d's that hit a target
key; walking forward turns each d back into a byte when the low byte x of the running hash keeps x + d in
0..255 (then b = x ^ (x + d) and nothing carries).  Each solve fixes a few random prefix bytes, so a seeded
random.Random makes the search, and what it finds, repeatable.

    python tools/fnv_preimage.py <key hex> [seed]
"""
from __future__ import annotations

import random
import sys

BASIS = 0xCBF29CE484222325
PRIME = 0x100000001B3
MASK = (1 << 64) - 1


def fnv1a64(data: bytes) -> int:
    h = BASIS
    for b in data:
        h = ((h ^ b) * PRIME) & MASK
    return h


def addr_bytes(u: int, l: int) -> bytes:
    return u.to_bytes(8, "little") + l.to_bytes(8, "little")


def addr_key(u: int, l: int) -> int:
    return fnv1a64(addr_bytes(u, l))


def lll(b: list[list[int]], num: int = 99, den: int = 100) -> list[list[int]]:
    """Integral LLL (H. Cohen, A Course in Computational Algebraic Number Theory, Alg. 2.6.7), exact
    integers only, Lovasz constant num/den.  The rows of b must be independent; b is reduced in place."""
    n = len(b)
    dot = lambda x, y: sum(p * q for p, q in zip(x, y))  # noqa: E731
    d = [1] + [0] * n                     # d[i+1]: Gram determinant of the first i+1 rows
    lam = [[0] * n for _ in range(n)]

    def red(k, l_):
        if 2 * abs(lam[k][l_]) > d[l_ + 1]:
            q = (2 * lam[k][l_] + d[l_ + 1]) // (2 * d[l_ + 1])
            b[k] = [x - q * y for x, y in zip(b[k], b[l_])]
            lam[k][l_] -= q * d[l_ + 1]
            for i in range(l_):
                lam[k][i] -= q * lam[l_][i]

    def swap(k, kmax):
        b[k], b[k - 1] = b[k - 1], b[k]
        for j in range(k - 1):
            lam[k][j], lam[k - 1][j] = lam[k - 1][j], lam[k][j]
        la = lam[k][k - 1]
        bb = (d[k - 1] * d[k + 1] + la * la) // d[k]
        for i in range(k + 1, kmax + 1):
            t = lam[i][k]
            lam[i][k] = (d[k + 1] * lam[i][k - 1] - la * t) // d[k]
            lam[i][k - 1] = (bb * t + la * lam[i][k]) // d[k + 1]
        d[k] = bb

    d[1] = dot(b[0], b[0])
    k, kmax = 1, 0
    while k < n:
        if k > kmax:
            kmax = k
            for j in range(k + 1):
                u = dot(b[k], b[j])
                for i in range(j):
                    u = (d[i + 1] * u - lam[k][i] * lam[j][i]) // d[i]
                if j < k:
                    lam[k][j] = u
                else:
                    d[k + 1] = u
                    assert u != 0, "dependent rows"
        red(k, k - 1)
        if den * d[k + 1] * d[k - 1] < num * d[k] * d[k] - den * lam[k][k - 1] ** 2:
            swap(k, kmax)
            k = max(1, k - 1)
        else:
            for l_ in range(k - 2, -1, -1):
                red(k, l_)
            k += 1
    return b


def _bytes_of(prefix: bytes, ds: list[int]) -> bytes | None:
    """The bytes after `prefix` whose steps add ds to the running hash, or None if one would carry."""
    h = fnv1a64(prefix)
    out = bytearray(prefix)
    for dv in ds:
        x = h & 0xFF
        if not 0 <= x + dv <= 255:
            return None
        out.append(x ^ (x + dv))
        h = ((h + dv) * PRIME) & MASK
    return bytes(out)


def _solve(prefix: bytes, target: int) -> list[bytes]:
    """Every 16-byte preimage of `target` starting with `prefix` that the reduced lattice offers."""
    m = 16 - len(prefix)
    coef = [pow(PRIME, m - j, 1 << 64) for j in range(m)]          # of d for free byte j
    rhs = (target - fnv1a64(prefix) * pow(PRIME, m, 1 << 64)) & MASK
    big, emb = 1 << 80, 64                                           # constraint weight, embedding
    rows = [[int(i == j) for i in range(m)] + [big * coef[j], 0] for j in range(m)]
    rows.append([0] * m + [big << 64, 0])
    rows.append([0] * m + [-big * rhs, emb])
    red = lll(rows)
    kernel = [r[:m] for r in red if r[m] == 0 and r[m + 1] == 0]
    found = []
    for r in red:
        if r[m] != 0 or abs(r[m + 1]) != emb:
            continue
        base = [x if r[m + 1] == emb else -x for x in r[:m]]
        cands = [base] + [[x + s * y for x, y in zip(base, k)] for k in kernel for s in (1, -1)]
        for ds in cands:
            out = _bytes_of(prefix, ds)
            if out is not None and fnv1a64(out) == target:
                found.append(out)
    return found


def preimages(target: int, count: int, seed: int, prefix_len: int = 3, avoid=()) -> list[tuple[int, int]]:
    """`count` distinct addresses (u, l) with FNV-1a key `target`, none of them in `avoid`, found from
    random prefixes of `prefix_len` bytes drawn from random.Random(seed)."""
    rng = random.Random(seed)
    seen = {addr_bytes(u, l) for u, l in avoid}
    out = []
    while len(out) < count:
        prefix = bytes(rng.randrange(256) for _ in range(prefix_len))
        for raw in sorted(_solve(prefix, target)):
            if raw not in seen and len(out) < count:
                seen.add(raw)
                out.append((int.from_bytes(raw[:8], "little"), int.from_bytes(raw[8:], "little")))
    return out


if __name__ == "__main__":
    key = int(sys.argv[1], 16)
    for u, l in preimages(key, 2, int(sys.argv[2]) if len(sys.argv) > 2 else 1):
        print(f"u={u:#018x} l={l:#018x} key={addr_key(u, l):#018x}")
