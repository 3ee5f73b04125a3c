"""GPU tests of the attention backward's head-sized last slice and of its query-tile loop (`pytest -m gpu`).

The last output slice runs its MMAs at N = min(64, d - col0), and the dQ columns of a slice are split between the two warpgroups
(24 + 16 for d = 40), so warpgroup 1 reads K starting 16, 32, 48 or 64 bytes into its swizzle rows: the head dims below reach every
slice width 8 ... 64 and every such offset.  The query-tile loop of a CTA walks 1, 2, 3 or more tiles, set by Lq, by the query split
(whole 128-row units per split, the last one possibly shorter) and, for causal attention, by the diagonal (a CTA of kv tile kt
starts at query tile 2 kt).  dQ / dK / dV are checked against float64 with tests/kernel_check.py's GRAD bounds, and written into
canary buffers.

Query splits below are those of a 132-SM H100 (plan_qsplit in attention.cu: a split when the (kv tile, head, image) CTAs fill less
than 4/5 of the SMs).
"""
import pytest
import torch

from kernel_check import GRAD, compare
from test_gpu_clip import GRAD_CAUSAL_DK, causal_ref, problem, run_causal
from test_gpu_edges import AttnProblem, check_attention, rnd

pytestmark = pytest.mark.gpu

DEV = "cuda"

# (B, H, Lq, Lkv, d, fused, pad): query tiles per CTA
TILE_CASES = [
    (2, 3, 50, 300, 40, False, 8),        # 1 tile (50 rows), 3 kv tiles
    (2, 3, 100, 200, 48, False, 0),       # 2 tiles, the second part-filled
    (1, 112, 160, 96, 40, False, 64),     # 3 tiles, no split (112 CTAs), Lkv not a multiple of 64
    (1, 112, 300, 130, 56, False, 0),     # 5 tiles, no split, Lkv = 128 + 2
    (1, 128, 64, 64, 64, True, 0),        # 1 full tile, no split
    (1, 3, 700, 200, 40, False, 8),       # split: 2 tiles per CTA, the last split 1 tile (700 = 10 * 64 + 60)
    (1, 40, 2470, 100, 72, False, 0),     # split: 6 tiles per CTA, the last split 3 (the last part-filled); slices 64 + 8
    (1, 2, 4096, 4096, 40, True, 0),      # config 2's self-attention shape, 2 heads: a 5-way split, 14 tiles per CTA, the last 8
]


@pytest.mark.parametrize("B,H,Lq,Lkv,d,fused,pad", TILE_CASES)
def test_attn_bwd_query_tiles(B, H, Lq, Lkv, d, fused, pad):
    check_attention(AttnProblem(B, H, Lq, Lkv, d, fused, pad), f"attn B{B} H{H} Lq{Lq} Lkv{Lkv} d{d}")


# every last-slice width 8 ... 64 with one, two and three 64-column boxes per head row
HEAD_DIMS = [8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 96, 112, 120, 136, 160, 176, 184]


@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("split", [False, True])
def test_attn_bwd_slice_widths(d, split):
    # split: 1 x 2 heads x 2 kv tiles -> a two-way query split, 2 tiles per CTA; else 112 heads, 3 query tiles per CTA
    B, H, Lq, Lkv = (1, 2, 200, 150) if split else (1, 112, 190, 70)
    check_attention(AttnProblem(B, H, Lq, Lkv, d, False, 8, seed=d), f"attn d{d} split{int(split)}")


def test_attn_bwd_kv_bias_mask():
    """An additive kv bias with a masked (-inf) key range that covers whole 64-row dS tiles of one warpgroup and a ragged part of
    another, on a 3-tile, unsplit problem."""
    B, H, Lq, Lkv, d = 2, 64, 150, 250, 40
    bias = (torch.randn(B, Lkv, generator=torch.Generator().manual_seed(7)) * 2.0).to(DEV)
    bias[0, 60:200] = -float("inf")
    bias[1, :70] = -float("inf")
    check_attention(AttnProblem(B, H, Lq, Lkv, d, False, 0, bias=bias), "attn kv_bias mask")


# causal (B, H, L, d): B * H * ceil(L / 128) >= 106 gives no split, so the CTA of kv tile kt walks ceil(L / 64) - 2 kt tiles (1, 3
# and 5 at L = 320; 2 and 4 at L = 200); the others split the query range, and splits that end above their kv tile exit
CAUSAL_CASES = [(1, 36, 320, 40), (1, 36, 320, 64), (1, 54, 200, 80), (2, 3, 65, 40), (2, 3, 600, 40), (1, 4, 1000, 56)]


@pytest.mark.parametrize("B,H,L,d", CAUSAL_CASES)
def test_attn_bwd_causal_tiles(B, H, L, d):
    q, k, v, bias, do = problem(B, H, L, d, True, seed=11)
    name = f"causal B{B} H{H} L{L} d{d}"
    _, _, (dq, dk, dv), g = run_causal(q, k, v, bias, do)
    _, _, dq_ref, dk_ref, dv_ref = causal_ref(q, k, v, bias, do.view(B, L, H, d))
    for nm, got, ref, rows in (("dQ", dq, dq_ref, 64), ("dK", dk, dk_ref, 128), ("dV", dv, dv_ref, 128)):
        compare(f"{name} {nm}", got.reshape(B, L, H * d), ref.reshape(B, L, H * d), GRAD_CAUSAL_DK if nm == "dK" else GRAD,
                block=(rows, d))
    g.check(f"{name} gradients")


def _bwd_bits(p: AttnProblem, o, lse, do):
    (dq, dk, dv), cans = p.backward(o, lse, do)
    return [c.buf.view(torch.int16).clone() for c in cans]


@pytest.mark.parametrize("B,H,Lq,Lkv,d", [(1, 8, 256, 256, 40), (2, 64, 200, 256, 72), (1, 4, 77, 77, 80)])
def test_attn_bwd_bit_identical_repeats(B, H, Lq, Lkv, d):
    """Lkv <= 256: at most two CTAs add into a dQ element, and a two-way query split (1 x 8 heads x 2 kv tiles) gives two dK / dV
    partials; both are order-independent fp32 sums, so repeats agree bit for bit."""
    p = AttnProblem(B, H, Lq, Lkv, d, False, 0, seed=3)
    o, lse = p.forward()
    do = rnd(B, Lq, H * d, seed=98)
    first = _bwd_bits(p, o, lse, do)
    for _ in range(3):
        again = _bwd_bits(p, o, lse, do)
        assert all(torch.equal(a, f) for a, f in zip(again, first)), "backward changed on a repeated call"


@pytest.mark.parametrize("L,d", [(77, 40), (256, 40), (77, 80)])
def test_attn_bwd_causal_bit_identical_repeats(L, d):
    q, k, v, bias, do = problem(2, 3, L, d, True, seed=13)
    first = run_causal(q, k, v, bias, do)[3].buf.view(torch.int16).clone()
    for _ in range(3):
        assert torch.equal(run_causal(q, k, v, bias, do)[3].buf.view(torch.int16), first)
