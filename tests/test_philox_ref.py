"""The numpy Philox4x32-10 of tests/philox_ref.py against the known-answer vectors published with Random123 (kat_vectors), and the
dropout mask restated from it on properties that need no GPU."""
import numpy as np

from philox_ref import dropout_keep, philox4x32_10

KAT = [   # counter (4 words), key (2 words) -> output (4 words)
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


def test_philox4x32_10_known_answers():
    for ctr, key, want in KAT:
        got = tuple(int(w) for w in philox4x32_10(*ctr, *key))
        assert got == want, f"ctr {ctr} key {key}: {[hex(w) for w in got]} != {[hex(w) for w in want]}"


def test_philox_vectorised_matches_scalar():
    c = np.arange(5, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15 & 0xFFFFFFFF)
    batch = np.stack(philox4x32_10(c, c + 1, 7, 3, 0xDEADBEEF, 0x12345678), axis=1)
    for j in range(5):
        one = [int(w) for w in philox4x32_10(int(c[j]), int(c[j]) + 1, 7, 3, 0xDEADBEEF, 0x12345678)]
        assert [int(w) for w in batch[j]] == one


def test_dropout_keep_mask_properties():
    keep0 = dropout_keep(8, 64, 0.0, seed=1, draw=0, site=1)
    assert keep0.all()                                                       # p = 0 keeps everything (threshold 0)
    a = dropout_keep(64, 256, 0.5, seed=1, draw=0, site=1)
    assert abs(a.mean() - 0.5) < 0.02
    assert (a != dropout_keep(64, 256, 0.5, seed=1, draw=0, site=2)).mean() > 0.4     # another site: an independent mask
    hi = dropout_keep(64, 256, 0.5, seed=1, draw=1 << 32, site=1)            # draw_hi enters through the key
    assert (a != hi).mean() > 0.4
    assert (hi == dropout_keep(64, 256, 0.5, seed=1 ^ (1 << 32), draw=0, site=1)).all()   # ... exactly as seed_hi does
    assert abs(dropout_keep(64, 256, 0.999, seed=5, draw=0, site=1).mean() - (1 - 65470 / 65536)) < 2e-3
