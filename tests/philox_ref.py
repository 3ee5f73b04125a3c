"""Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC 2011) in numpy, and the keep mask
of hcp_dropout_bf16 restated from it.

Arithmetic is uint64 masked to 32 bits, so the 32x32 -> 64-bit products are exact.  Every function takes arrays of counters and
returns arrays of the same shape, so a whole mask is one call.
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)
S32 = np.uint64(32)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Ten rounds on counter (c0, c1, c2, c3) with key (k0, k1); arguments are broadcastable integer arrays (values < 2^32).
    Returns four uint64 arrays holding the 32-bit output words."""
    c0, c1, c2, c3, k0, k1 = (np.asarray(a, dtype=np.uint64) & MASK for a in (c0, c1, c2, c3, k0, k1))
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2                          # < 2^64: exact in uint64
        hi0, lo0 = p0 >> S32, p0 & MASK
        hi1, lo1 = p1 >> S32, p1 & MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def dropout_keep(rows: int, ncols: int, p: float, seed: int, draw: int, site: int) -> np.ndarray:
    """bool [rows, ncols]: the elements hcp_dropout_bf16 keeps for state = (seed, draw) and `site` over a column range of width
    ncols (% 8 == 0).  Vector i = r * (ncols / 8) + c / 8 draws Philox with counter (i_lo, i_hi, site, draw_lo) and key
    (seed_lo, seed_hi ^ draw_hi); element k of the vector is kept when the 16-bit half k % 2 of word k / 2 is >= (uint32)(p * 65536),
    the product taken in fp32 as the kernel does."""
    assert ncols % 8 == 0
    i = np.arange(rows * (ncols // 8), dtype=np.uint64)
    words = philox4x32_10(i & MASK, i >> S32, site, draw & 0xFFFFFFFF, seed & 0xFFFFFFFF, ((seed >> 32) ^ (draw >> 32)) & 0xFFFFFFFF)
    w = np.stack(words, axis=1)                                             # [vectors, 4]
    halves = np.stack([w & np.uint64(0xFFFF), w >> np.uint64(16)], axis=2)  # [vectors, 4, 2]: element 2j (low half), 2j + 1 (high)
    thr = np.uint64(int(np.float32(p) * np.float32(65536.0)))
    return (halves >= thr).reshape(rows, ncols)
