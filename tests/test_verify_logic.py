"""The group-split EF128 that the verified gets compute (fingerprint.cuh: ef_group_sum, ef_group_finish),
restated in numpy and compared with the oracle's serial EF128 (oracle/fingerprint.c).

Inside a 16-stripe group the absorb step only adds to each lane's (a, b), so lane l's sums over a group
can be taken apart from the chain and added in afterwards, followed by the group's scramble.  This is
the algebra k_get_small relies on when its 16 warps fingerprint a page in shared memory at once."""
import numpy as np
import pytest

M64 = (1 << 64) - 1


def _secret(i: int) -> int:
    z = (0x4544474546555345 + (i + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


S = np.array([_secret(i) for i in range(128)], dtype=np.uint64).reshape(32, 4)


def _fold(x: int, y: int) -> int:
    p = x * y
    return (p & M64) ^ (p >> 64)


def _av(h: int) -> int:
    h ^= h >> 37
    h = (h * 0x165667919E3779F9) & M64
    return h ^ (h >> 32)


def group_sums(data: np.ndarray) -> np.ndarray:
    """[groups, 32, 2] uint64: lane l's sums {A, B} over each 16-stripe group (bytes >= n read as zero)."""
    n = len(data)
    stripes = (n + 511) // 512
    groups = (stripes + 15) // 16
    buf = np.zeros(groups * 16 * 512, dtype=np.uint8)
    buf[:n] = data
    x = buf.view("<u8").reshape(groups * 16, 32, 2)
    x[stripes:] = 0                                     # stripes past the page absorb nothing
    x0, x1 = x[..., 0], x[..., 1]
    d0, d1 = x0 ^ S[:, 0], x1 ^ S[:, 1]
    m32 = np.uint64(0xFFFFFFFF)
    with np.errstate(over="ignore"):
        fa = (d0 & m32) * (d0 >> np.uint64(32)) + x1
        fb = (d1 & m32) * (d1 >> np.uint64(32)) + x0
    fa[stripes:] = 0
    fb[stripes:] = 0
    # sums mod 2^64 (numpy's uint64 adds wrap)
    A = np.add.reduce(fa.reshape(groups, 16, 32), axis=1, dtype=np.uint64)
    B = np.add.reduce(fb.reshape(groups, 16, 32), axis=1, dtype=np.uint64)
    return np.stack([A, B], axis=-1)


def group_finish(sums: np.ndarray, n: int) -> tuple[int, int]:
    """The one-warp chain: add each group's sums, scramble after every group that reaches its 16th
    stripe, then fold the 32 lanes."""
    stripes = (n + 511) // 512
    full = stripes // 16
    U, V = (n * 0x9E3779B185EBCA87) & M64, (~(n * 0xC2B2AE3D27D4EB4F)) & M64
    for lane in range(32):
        s0, s1, s2, s3 = (int(v) for v in S[lane])
        a, b = s2, s3
        for g in range(len(sums)):
            a = (a + int(sums[g, lane, 0])) & M64
            b = (b + int(sums[g, lane, 1])) & M64
            if g < full:
                a = (((a ^ (a >> 47)) ^ s2) * 0x9E3779B1) & M64
                b = (((b ^ (b >> 47)) ^ s3) * 0x85EBCA77) & M64
        U = (U + _fold(a ^ s0, b ^ s1)) & M64
        V = (V + _fold(a ^ s3, b ^ s2)) & M64
    return _av(V), _av(U)


def _page(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


LENGTHS = ([1 << k for k in range(6, 21)]
           + [8192 - 8, 8192 + 100, 3 * 8192 + 512 + 7, 512 * 17 + 1, 65536 - 300, 131072 - 16, 1000, 40])


@pytest.mark.parametrize("n", LENGTHS)
def test_group_split_matches_the_serial_fingerprint(oracle, n):
    for seed in (1, 2):
        page = _page(n, seed * 1000 + n)
        want = oracle.fingerprint128(page)
        assert group_finish(group_sums(page), n) == tuple(want), (n, seed)


def test_group_split_sees_one_flipped_byte(oracle):
    page = _page(65536, 7)
    good = group_finish(group_sums(page), 65536)
    page[40000] ^= 0x10
    assert group_finish(group_sums(page), 65536) != good
    assert tuple(oracle.fingerprint128(page)) != good
