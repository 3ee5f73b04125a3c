"""GPU tests of the sm_90a kernels at the edges of their tilings (`pytest -m gpu`).

Every kernel picks its tiling from the problem shape: the GEMM its column-tile width BN (32 / 64 / 128 / 160 / 176) and how many
K-splits to run, the convolution its pixel box (one row of 128 pixels for maps >= 128 wide, several images per tile for tiny maps),
the attention its kv tile (64 rows for head dims > 128) and how far to split the query range in the backward.  The cases below
reach each of those choices with ragged tails, against float64 references (tests/kernel_check.py: global, per-tile and max-abs
errors), and write every output of a direct C-ABI call into a canary buffer whose surroundings must stay untouched.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import FWD, GRAD, LORA, LSE_ABS, Canary, compare
from lora_conv_plan import tile_n

pytestmark = pytest.mark.gpu

from hcp_diffusion_b200 import _lib, ops  # noqa: E402
from hcp_diffusion_b200._lib import AttnArgs, AttnBwdArgs, HcpError, call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402,F401  (runtime and models import each other: models first)
from hcp_diffusion_b200.ops import ConvPack, LinearPack, LoraBlockRef  # noqa: E402
from hcp_diffusion_b200.runtime import pack_lora  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


def as_pack_group(pack):
    class G:
        pass
    g = G()
    g.pack = pack
    return g


# ----------------------------------------------------------------------------------------------------------------------
# GEMM: out = x . W^T + bias + rowbias + residual through hcp_gemm_bf16
# ----------------------------------------------------------------------------------------------------------------------
def gemm_case(M, K, N, seed=0, rows_per_group=77):
    x = rnd(M, K, seed=seed + 1)
    w = rnd(N, K, scale=1 / math.sqrt(K), seed=seed + 2)
    bias = rnd(N, seed=seed + 3, dtype=torch.float32)
    rb = rnd((M + rows_per_group - 1) // rows_per_group, N, scale=0.5, seed=seed + 4, dtype=torch.float32)
    res_buf = rnd(M, N + 16, seed=seed + 5)                     # residual pitch ldr = N + 16 != N
    res = res_buf[:, :N]
    ref = x.to(F64) @ w.to(F64).t() + bias.to(F64) + rb.to(F64).repeat_interleave(rows_per_group, 0)[:M] + res.to(F64)
    return x, w, bias, rb, res, ref


def run_gemm(x, w, bias, rb, res, rows_per_group, out):
    M, K = x.shape
    N = w.shape[0]
    ops.gemm_raw([(x, K, K)], [(w, K, N, 0)], M, N, out.view, out.ld, bias=bias, rowbias=rb, rows_per_group=rows_per_group,
                 residual=res, ldr=res.stride(0))


# A ragged last column tile in every BN instantiation (N 8 and 24: BN 32; 40 and 192: 64; 200: 128; 336: 176, the 320 + 16
# rank-rows case; 2560: 160), M tails (one row; 63 rows, where the second MMA warpgroup has no valid row; 65; 129), K tails (a partial
# last k-block of 1..3 k-steps) and a persistent walk with far more work items than SMs (the producer runs ahead across work items)
GEMM_CASES = [(300, 320, 8), (300, 320, 24), (300, 320, 40), (300, 320, 192), (300, 320, 200), (300, 320, 336), (300, 320, 2560),
              (1, 320, 320), (63, 320, 336), (65, 320, 200), (129, 320, 40),
              (200, 8, 64), (200, 40, 200), (200, 72, 336), (200, 1000, 24),
              (8192, 320, 2560)]


@pytest.mark.parametrize("M,K,N", GEMM_CASES)
def test_gemm_tails(M, K, N):
    x, w, bias, rb, res, ref = gemm_case(M, K, N)
    out = Canary(M, N)
    run_gemm(x, w, bias, rb, res, 77, out)
    compare(f"gemm M{M} K{K} N{N}", out.view, ref, FWD, block=(128, tile_n(N)))
    out.check("gemm out")


def test_gemm_three_segments_with_kblock_major_operand():
    """cat(x1, x2) . W^T + T . Bl^T: three K-segments (640 + 320 + a rank-20 LoRA segment, 2 of 4 k-steps in its only k-block), the
    first B operand k-block-major [K/64][N][64]."""
    M, N, r = 300, 320, 20
    x1, x2 = rnd(M, 640, seed=1), rnd(M, 320, seed=2)
    w = rnd(N, 960, scale=1 / math.sqrt(960), seed=3)
    t = torch.zeros(M, 64, dtype=BF, device=DEV)
    t[:, :r] = rnd(M, r, seed=4)
    bl = torch.zeros(N, 64, dtype=BF, device=DEV)
    bl[:, :r] = rnd(N, r, scale=0.3, seed=5)
    bias = rnd(N, seed=6, dtype=torch.float32)
    w_tiled = ops.tile_kmajor(w[:, :640].contiguous())
    out = Canary(M, N)
    ops.gemm_raw([(x1, 640, 640), (x2, 320, 320), (t, 64, r)], [(w_tiled, N, N, 0, True), (w, 960, N, 640), (bl, 64, N, 0)], M, N,
                 out.view, out.ld, bias=bias)
    ref = torch.cat([x1, x2, t[:, :r]], 1).to(F64) @ torch.cat([w, bl[:, :r]], 1).to(F64).t() + bias.to(F64)
    compare("gemm 3 segments", out.view, ref, FWD, block=(128, 160))
    out.check("gemm 3 segments")


# (M, K, N, splits): both branches of plan_splits -- two K halves when a third to a half of the SMs hold a tile, otherwise up to one
# wave of SMs -- and its cap of 16; M tails and a row-bias group of 77 rows that does not divide the 128-row tiles
SPLITK_CASES = [(1000, 2560, 1280, 2), (200, 1280, 1280, 5), (100, 8192, 640, 16)]


@pytest.mark.parametrize("M,K,N,splits", SPLITK_CASES)
def test_gemm_split_k(M, K, N, splits, monkeypatch):
    lib = _lib.lib()
    assert lib.hcp_splitk_workspace_bytes(M, N, K) == splits * M * N * 4
    x, w, bias, rb, res, ref = gemm_case(M, K, N, seed=10)
    out = Canary(M, N)
    run_gemm(x, w, bias, rb, res, 77, out)
    compare(f"split-K x{splits} M{M} K{K} N{N}", out.view, ref, FWD, block=(128, tile_n(N)))
    out.check("split-K out")
    again = Canary(M, N)
    run_gemm(x, w, bias, rb, res, 77, again)
    assert torch.equal(again.view.view(torch.int16), out.view.view(torch.int16)), "split-K result changed on a repeated call"
    monkeypatch.setattr(lib, "hcp_splitk_workspace_bytes", lambda *a: 0)          # no workspace: the same GEMM unsplit
    whole = Canary(M, N)
    run_gemm(x, w, bias, rb, res, 77, whole)
    compare(f"split-K x{splits} vs unsplit", out.view, whole.view.to(F64), FWD, block=(128, tile_n(N)))


# ----------------------------------------------------------------------------------------------------------------------
# 3x3 convolution: forward (mode 0) and input gradient (stride 1: mode 0 with flipped taps; stride 2: mode 1) via hcp_conv3x3_bf16
# ----------------------------------------------------------------------------------------------------------------------
# (B, H, W, Cin, Cout, stride)
CONV_CASES = [
    (1, 128, 128, 320, 320, 1), (1, 128, 128, 320, 320, 2),     # SDXL 1024 px top level: one-row 128-pixel boxes; its downsampler
    (1, 4, 256, 64, 64, 1), (2, 4, 256, 64, 64, 2),             # two boxes per row; stride 2 to a 128-wide map (5-D box, bw 128)
    (2, 16, 64, 64, 64, 1), (2, 64, 16, 64, 64, 1), (1, 128, 8, 64, 64, 1), (1, 128, 8, 64, 64, 2),       # non-square maps
    (3, 4, 4, 64, 64, 1), (3, 2, 2, 64, 64, 1), (3, 1, 1, 64, 64, 1), (3, 2, 2, 64, 128, 2),              # a part-filled image tile
    (1, 16, 16, 64, 128, 1),                                     # two K-splits
    (1, 8, 8, 2560, 640, 1),
    (2, 16, 16, 64, 8, 1), (2, 16, 16, 64, 40, 1), (2, 16, 16, 64, 200, 2), (2, 16, 16, 64, 336, 1),      # Cout edges (no dgrad)
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", CONV_CASES)
def test_conv3x3_edges(B, H, W, Cin, Cout, stride):
    x = rnd(B, H * W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2, dtype=torch.float32)
    bias = rnd(Cout, scale=0.5, seed=3, dtype=torch.float32)
    rb = rnd(B, Cout + 8, scale=0.5, seed=4, dtype=torch.float32)[:, 4:4 + Cout]
    Ho, Wo = H // stride, W // stride
    M = B * Ho * Wo
    res = rnd(M, Cout, seed=5)
    pack = ConvPack(w, bias, stride)
    out = Canary(M, Cout, ld=Cout, col0=0)
    ops.conv3x3_raw(x, pack.W, B, H, W, Cin, Cout, stride, 0, out.view, bias=pack.bias, rowbias=rb, residual=res, rowbias_ld=rb.stride(0))
    xr = x.to(F64).view(B, H, W, Cin).permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.conv2d(xr, w.to(BF).to(F64), bias.to(F64), stride=stride, padding=1) + rb.to(F64)[:, :, None, None]
    yr = yr.permute(0, 2, 3, 1).reshape(M, Cout)
    compare(f"conv B{B} {H}x{W} {Cin}->{Cout} s{stride}", out.view, yr + res.to(F64), FWD, block=(128, tile_n(Cout)))
    out.check("conv out")
    if Cout % 64:
        return                                   # the input gradient reads Cout channels per pixel: 64-channel multiples only
    dy = rnd(M, Cout, seed=6)
    yr.backward(dy.to(F64))
    dx = Canary(B * H * W, Cin, ld=Cin, col0=0)
    if stride == 1:
        ops.conv3x3_raw(dy, pack.Wd, B, H, W, Cout, Cin, 1, 0, dx.view)
    else:
        ops.conv3x3_raw(dy, pack.Wd, B, Ho, Wo, Cout, Cin, 2, 1, dx.view)
    compare(f"conv dgrad B{B} {H}x{W} {Cin}->{Cout} s{stride}", dx.view, xr.grad.permute(0, 2, 3, 1).reshape(-1, Cin), FWD,
            block=(128, tile_n(Cin)))
    dx.check("conv dgrad")


# ----------------------------------------------------------------------------------------------------------------------
# attention through hcp_attn_fwd_bf16 / hcp_attn_bwd_bf16
# ----------------------------------------------------------------------------------------------------------------------
def attn_ref(q, k, v, bias, do):
    """float64 softmax(q k^T / sqrt(d) + bias) v, its natural-log logsumexp and the three input gradients, chunked over heads.
    q / do [B, Lq, H, d], k / v [B, Lkv, H, d], bias [B, Lkv] or None."""
    B, Lq, H, d = q.shape
    Lkv = k.shape[1]
    o, dq = torch.empty_like(q, dtype=F64), torch.empty_like(q, dtype=F64)
    dk, dv = torch.empty_like(k, dtype=F64), torch.empty_like(v, dtype=F64)
    lse = torch.empty(B, H, Lq, dtype=F64, device=q.device)
    step = max(1, (1 << 26) // (Lq * Lkv))
    for b in range(B):
        for h0 in range(0, H, step):
            hs = slice(h0, min(H, h0 + step))
            qh, kh, vh = (t[b, :, hs].to(F64).transpose(0, 1).requires_grad_(True) for t in (q, k, v))
            s = qh @ kh.transpose(-1, -2) / math.sqrt(d)
            if bias is not None:
                s = s + bias[b].to(F64)
            oh = torch.softmax(s, -1) @ vh
            oh.backward(do[b, :, hs].to(F64).transpose(0, 1))
            with torch.no_grad():
                o[b, :, hs] = oh.transpose(0, 1)
                lse[b, hs] = torch.logsumexp(s, -1)
            dq[b, :, hs], dk[b, :, hs], dv[b, :, hs] = (t.grad.transpose(0, 1) for t in (qh, kh, vh))
    return o, lse, dq, dk, dv


class AttnProblem:
    """q / k / v as column blocks of bf16 buffers: one fused [B, L, 3C + pad] QKV buffer (self-attention), or q in [B, Lq, C + pad]
    and k | v in [B, Lkv, 2C + pad] (cross-attention); pad > 0 gives a leading dimension larger than the data."""

    def __init__(self, B, H, Lq, Lkv, d, fused, pad, seed=0, q=None, k=None, v=None, bias=None):
        C_ = H * d
        self.B, self.H, self.Lq, self.Lkv, self.d, self.C, self.fused = B, H, Lq, Lkv, d, C_, fused
        q = rnd(B, Lq, H, d, seed=seed + 1) if q is None else q.to(BF)
        k = rnd(B, Lkv, H, d, seed=seed + 2) if k is None else k.to(BF)
        v = rnd(B, Lkv, H, d, seed=seed + 3) if v is None else v.to(BF)
        self.q, self.k, self.v, self.bias = q, k, v, bias
        if fused:
            assert Lq == Lkv
            self.qkv = torch.zeros(B, Lq, 3 * C_ + pad, dtype=BF, device=DEV)
            self.qkv[..., :3 * C_] = torch.cat([t.reshape(B, Lq, C_) for t in (q, k, v)], -1)
            base, ld = self.qkv.data_ptr(), self.qkv.shape[-1]
            self.ptrs = (base, ld, base + 2 * C_, ld, base + 4 * C_, ld)
        else:
            self.qb = torch.zeros(B, Lq, C_ + pad, dtype=BF, device=DEV)
            self.qb[..., :C_] = q.reshape(B, Lq, C_)
            self.kvb = torch.zeros(B, Lkv, 2 * C_ + pad, dtype=BF, device=DEV)
            self.kvb[..., :2 * C_] = torch.cat([k.reshape(B, Lkv, C_), v.reshape(B, Lkv, C_)], -1)
            ldq, ldkv = self.qb.shape[-1], self.kvb.shape[-1]
            self.ptrs = (self.qb.data_ptr(), ldq, self.kvb.data_ptr(), ldkv, self.kvb.data_ptr() + 2 * C_, ldkv)

    def forward(self):
        """-> (O canary [B*Lq, C] at ld C + 64, lse [B, H, Lq] fp32)"""
        o = Canary(self.B * self.Lq, self.C)
        lse = torch.full((self.B, self.H, self.Lq), float("nan"), dtype=torch.float32, device=DEV)
        a = AttnArgs()
        a.q, a.ldq, a.k, a.ldk, a.v, a.ldv = self.ptrs
        a.B, a.H, a.Lq, a.Lkv, a.d = self.B, self.H, self.Lq, self.Lkv, self.d
        a.scale = 1.0 / math.sqrt(self.d)
        a.kv_bias = None if self.bias is None else self.bias.data_ptr()
        a.o, a.ldo, a.lse = o.view.data_ptr(), o.ld, lse.data_ptr()
        call("hcp_attn_fwd_bf16", C.byref(a), stream_ptr())
        return o, lse

    def backward(self, o, lse, do):
        """-> dQ, dK, dV as [B, L, H, d] views of canary buffers laid out like the sources: one fused [B*L, 3C] rectangle, or dQ in
        [B*Lq, C] and dK | dV in [B*Lkv, 2C] (each at a leading dimension 64 larger), plus the canaries."""
        B, H, Lq, Lkv, d, C_ = self.B, self.H, self.Lq, self.Lkv, self.d, self.C
        if self.fused:
            g = Canary(B * Lq, 3 * C_)
            cans = [g]
            dq_p, dk_p, dv_p = g.view.data_ptr(), g.view.data_ptr() + 2 * C_, g.view.data_ptr() + 4 * C_
            lds = (g.ld, g.ld, g.ld)
            views = [g.view[:, i * C_:(i + 1) * C_] for i in range(3)]
        else:
            gq, gkv = Canary(B * Lq, C_), Canary(B * Lkv, 2 * C_)
            cans = [gq, gkv]
            dq_p, dk_p, dv_p = gq.view.data_ptr(), gkv.view.data_ptr(), gkv.view.data_ptr() + 2 * C_
            lds = (gq.ld, gkv.ld, gkv.ld)
            views = [gq.view, gkv.view[:, :C_], gkv.view[:, C_:]]
        lib = _lib.lib()
        wsb = lib.hcp_attn_bwd_workspace_bytes(B, H, Lq, Lkv, d)
        ws = torch.empty((wsb // 4,), dtype=torch.float32, device=DEV)
        a = AttnBwdArgs()
        a.q, a.ldq, a.k, a.ldk, a.v, a.ldv = self.ptrs
        a.o, a.ldo, a.dout, a.lddo = o.view.data_ptr(), o.ld, do.data_ptr(), C_
        a.B, a.H, a.Lq, a.Lkv, a.d = B, H, Lq, Lkv, d
        a.scale = 1.0 / math.sqrt(d)
        a.kv_bias = None if self.bias is None else self.bias.data_ptr()
        a.lse = lse.data_ptr()
        a.dq, a.lddq, a.dk, a.lddk, a.dv, a.lddv = dq_p, lds[0], dk_p, lds[1], dv_p, lds[2]
        a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
        call("hcp_attn_bwd_bf16", C.byref(a), stream_ptr())
        Ls = (Lq, Lkv, Lkv)
        return [vw.reshape(B, L, H, d) for vw, L in zip(views, Ls)], cans


def check_attention(p: AttnProblem, name: str, backward=True):
    B, H, Lq, Lkv, d = p.B, p.H, p.Lq, p.Lkv, p.d
    o, lse = p.forward()
    do = rnd(B, Lq, H * d, seed=99)
    o_ref, lse_ref, dq_ref, dk_ref, dv_ref = attn_ref(p.q, p.k, p.v, p.bias, do.view(B, Lq, H, d))
    # blocks: one head of 64 query rows (the forward's warpgroup tile) / 128 kv rows (the backward's CTA)
    compare(f"{name} O", o.view.reshape(B, Lq, H * d), o_ref.reshape(B, Lq, H * d), FWD, block=(64, d))
    o.check(f"{name} O")
    assert torch.isfinite(lse).all(), f"{name}: lse not written everywhere"
    lerr = float((lse.to(F64) - lse_ref).abs().max())
    print(f"[{name} lse] maxabs={lerr:.3e}")
    assert lerr <= LSE_ABS, f"{name}: lse off by {lerr:.3e}"
    if not backward:
        return
    (dq, dk, dv), cans = p.backward(o, lse, do)
    for nm, got, ref, rows in (("dQ", dq, dq_ref, 64), ("dK", dk, dk_ref, 128), ("dV", dv, dv_ref, 128)):
        L = got.shape[1]
        if Lkv == 1 and nm != "dV":
            # a softmax over one key is constant: dQ = dK = 0 exactly, and the kernel may leave only rounding noise of dP - delta
            # (measured 1.7e-7 of max|dV|)
            noise = float(got.to(F64).abs().max() / dv_ref.abs().max())
            print(f"[{name} {nm}] max|{nm}| / max|dV| = {noise:.3e}")
            assert noise <= 5e-7, f"{name}: {nm} should vanish, max|{nm}| / max|dV| = {noise:.3e}"
            continue
        compare(f"{name} {nm}", got.reshape(B, L, H * d), ref.reshape(B, L, H * d), GRAD, block=(rows, d))
    for c in cans:
        c.check(f"{name} gradients")


# (B, H, Lq, Lkv, d, fused QKV buffer, ld padding)
ATTN_CASES = [
    (2, 2, 129, 129, 8, True, 0), (1, 3, 65, 231, 16, False, 64), (1, 2, 257, 64, 72, False, 0), (1, 2, 129, 257, 128, False, 64),
    (1, 2, 65, 154, 136, False, 0), (1, 2, 1, 1, 192, False, 0), (1, 2, 300, 300, 192, True, 64), (2, 3, 1, 129, 40, False, 8),
    # SDXL (head dim 64 at every level): 64x64 latent self- and 77-token cross-attention, and the 32x32 level's 20 heads
    (2, 10, 4096, 4096, 64, True, 0), (2, 10, 4096, 77, 64, False, 0), (1, 20, 1024, 1024, 64, True, 64),
    # backward query splits on a 132-SM H100: two (order-independent dK / dV partials), 32 (fp32 partial sums of dK / dV)
    (1, 8, 256, 256, 64, True, 0), (1, 2, 4096, 256, 80, False, 0),
    # dQ split by output column between the two warpgroups (32-column slices): d 96 (three full slices), 112 / 176 (a part-filled
    # warpgroup-1 half after the first slice), 160 (SD1.5's deepest head dim: warpgroup 1 has no column in the third slice) at a
    # query-split shape and as a 77-token cross-attention
    (1, 2, 200, 200, 96, False, 0), (1, 2, 257, 257, 112, True, 64), (1, 8, 256, 256, 160, True, 0), (2, 4, 300, 77, 160, False, 8),
    (1, 2, 129, 77, 176, False, 0),
]


@pytest.mark.parametrize("B,H,Lq,Lkv,d,fused,pad", ATTN_CASES)
def test_attention_edges(B, H, Lq, Lkv, d, fused, pad):
    check_attention(AttnProblem(B, H, Lq, Lkv, d, fused, pad), f"attn B{B} H{H} Lq{Lq} Lkv{Lkv} d{d}")


@pytest.mark.parametrize("d", [64, 128, 160])
@pytest.mark.parametrize("kind", ["large_logits", "masked_first_tile", "one_key"])
def test_attention_online_softmax_stress(kind, d):
    """Scores spanning about +-30 with a planted row maximum (~+45) in the first kv tile for odd query rows and in the last for even
    ones (the running max moves late: O and l must be rescaled); a -inf bias over the whole first kv tile (rows with no finite
    score yet); a bias that leaves one key (softmax = one-hot).  The backward is checked for the masked tile only: with a (nearly)
    one-hot softmax dQ and dK are differences of nearly equal numbers, which no bf16 kernel resolves."""
    B, H, Lq, Lkv = 1, 2, 130, 300
    k = torch.randn(B, Lkv, H, d, generator=torch.Generator().manual_seed(1)).to(DEV)
    q = torch.randn(B, Lq, H, d, generator=torch.Generator().manual_seed(2)).to(DEV)
    bias = None
    if kind == "large_logits":
        j = torch.where(torch.arange(Lq, device=DEV) % 2 == 1, 3, Lkv - 5)          # the planted key of each query row
        q = q * 7.0 + k[:, j] * (45 / math.sqrt(d))
    elif kind == "masked_first_tile":
        bias = torch.zeros(B, Lkv, device=DEV)
        bias[:, :128] = -float("inf")
    else:
        bias = torch.full((B, Lkv), -float("inf"), device=DEV)
        bias[:, 200] = 0.0
    check_attention(AttnProblem(B, H, Lq, Lkv, d, False, 0, q=q, k=k, bias=bias), f"attn stress {kind} d{d}",
                    backward=kind == "masked_first_tile")


# ----------------------------------------------------------------------------------------------------------------------
# LoRA layouts through LinearPack / pack_lora (K-segment and merged forms)
# ----------------------------------------------------------------------------------------------------------------------
# hosts: ranks of the blocks stacked on each host of a fused group (host i owns output rows [i*n, (i+1)*n)); k_splits: widths of the
# concatenated inputs
LORA_CASES = {
    "r20x3": ([(20,), (20,), (20,)], [320]),               # three blocks in one 64-column slab
    "r40x3": ([(40,), (40,), (40,)], [320]),               # slab-alignment gaps: columns 0-39, 64-103, 128-167
    "r64": ([(64,)], [320]),
    "r80": ([(80,)], [320]),                                # one block over two slabs (never merged: ranks sum above 64)
    "r128": ([(128,)], [640]),
    "r4x9": ([(4, 4, 4), (4, 4, 4), (4, 4, 4)], [320]),     # nine blocks in one slab: two launches of the gradient kernel
    "two_inputs": ([(20,)], [640, 320]),                    # the up-block conv_shortcut on the concatenated skip
}


@pytest.mark.parametrize("merge", [False, True])
@pytest.mark.parametrize("case", list(LORA_CASES))
def test_lora_layouts(case, merge):
    hosts, ks = LORA_CASES[case]
    M, n, alpha = 300, 320, 0.5
    K = sum(ks)
    N = n * len(hosts)
    W = rnd(N, K, scale=1 / math.sqrt(K), seed=1, dtype=torch.float32)
    b = rnd(N, scale=0.1, seed=2, dtype=torch.float32)
    pack = LinearPack(W, b, k_splits=ks if len(ks) > 1 else None)
    refs, per_host, seed = [], [], 10
    for i, ranks in enumerate(hosts):
        mine = []
        for r in ranks:
            down = rnd(r, K, scale=1 / math.sqrt(K), seed=seed, dtype=torch.float32).requires_grad_(True)
            up = rnd(n, r, scale=0.3, seed=seed + 1, dtype=torch.float32).requires_grad_(True)
            seed += 2
            mine.append(LoraBlockRef(down, up, alpha, i * n))
        refs += mine
        per_host.append((W[i * n:(i + 1) * n].contiguous(), i * n, n, mine))
    pack.attach_lora(refs)
    if merge:
        assert pack.enable_merge(per_host) == all(sum(r) <= 64 and len(r) <= 4 for r in hosts)
    pack_lora([as_pack_group(pack)])
    xs = [rnd(M, k, seed=3 + j).requires_grad_(True) for j, k in enumerate(ks)]
    y = ops.fused_linear(pack, xs)
    dy = rnd(M, N, seed=7)
    y.backward(dy)
    # float64 reference: y = x (W + sum alpha W_up W_down)^T + b on the bf16 inputs and the bf16 host weight
    xr = [x.detach().to(F64).requires_grad_(True) for x in xs]
    fac = [(blk.w_down.detach().to(F64).requires_grad_(True), blk.w_up.detach().to(F64).requires_grad_(True)) for blk in refs]
    Wp = W.to(BF).to(F64)
    delta = torch.zeros_like(Wp)
    for blk, (d_, u_) in zip(refs, fac):
        delta[blk.o0:blk.o0 + n] += alpha * (u_ @ d_)
    yr = torch.cat(xr, 1) @ (Wp + delta).t() + b.to(F64)
    yr.backward(dy.to(F64))
    compare(f"lora {case} merge={merge} y", y, yr.detach(), FWD)
    for j, (x, x_r) in enumerate(zip(xs, xr)):
        compare(f"lora {case} merge={merge} dx{j}", x.grad, x_r.grad, FWD)
    for i, (blk, (d_, u_)) in enumerate(zip(refs, fac)):
        off = 0
        for j, k in enumerate(ks):                               # W_down's gradient per input column range
            compare(f"lora {case} merge={merge} dW_down[{i}] cols {off}:{off + k}", blk.w_down.grad[:, off:off + k], d_.grad[:, off:off + k],
                    LORA, block=(64, 128))
            off += k
        compare(f"lora {case} merge={merge} dW_up[{i}]", blk.w_up.grad, u_.grad, LORA, block=(128, 64))


# ----------------------------------------------------------------------------------------------------------------------
# determinism and clean rejection
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gemm", "split_k", "conv", "attn_fwd", "attn_bwd"])
def test_repeated_call_is_bit_identical(kind):
    """The forward kernels have no floating-point atomics, and split-K sums its partials in a fixed order: a repeated call gives the
    same bits.  The attention backward reduces dQ with one fp32 red.add per 128-row kv tile and, when the query range is split,
    dK / dV through fp32 partials: with at most two kv tiles and at most two query splits every sum has two addends, so its result
    does not depend on their order.  Not asserted (they are not order-independent): the backward for longer kv ranges or more query
    splits, and the atomics-based LoRA / weight gradients."""
    def bits(*ts):
        return [t.contiguous().view(torch.int16 if t.dtype == BF else torch.int32).clone() for t in ts]

    if kind in ("gemm", "split_k"):
        M, K, N = (300, 320, 336) if kind == "gemm" else (100, 4096, 640)
        x, w, bias, rb, res, _ = gemm_case(M, K, N)
        runs = []
        for _ in range(2):
            out = Canary(M, N)
            run_gemm(x, w, bias, rb, res, 77, out)
            runs.append(bits(out.view))
    elif kind == "conv":
        B, H, Cin, Cout = 3, 16, 64, 128               # two K-splits
        x = rnd(B, H * H, Cin, seed=1)
        pack = ConvPack(rnd(Cout, Cin, 3, 3, scale=0.05, seed=2, dtype=torch.float32), None, 1)
        runs = []
        for _ in range(2):
            out = torch.empty(B, H * H, Cout, dtype=BF, device=DEV)
            ops.conv3x3_raw(x, pack.W, B, H, H, Cin, Cout, 1, 0, out)
            runs.append(bits(out))
    else:
        # Lkv = 256 (two kv tiles), Lq = 256 with B 1, H 8: the backward splits the query range in two
        p = AttnProblem(1, 8, 256, 256, 64, True, 0)
        do = rnd(1, 256, 512, seed=5)
        runs = []
        for _ in range(2):
            o, lse = p.forward()
            if kind == "attn_fwd":
                runs.append(bits(o.view, lse))
            else:
                runs.append(bits(*p.backward(o, lse, do)[0]))
    assert all(torch.equal(a, b) for a, b in zip(*runs)), f"{kind}: a repeated call changed the result"


def test_unsupported_shapes_raise_before_any_launch():
    """A 64x96 latent (SD1.5 at 512x768), head dim 200 and N % 8 != 0 are rejected with HcpError; nothing is launched."""
    before = _lib.launch_count
    x = torch.zeros(1, 64 * 96, 64, dtype=BF, device=DEV)
    pack = ConvPack(torch.zeros(64, 64, 3, 3, device=DEV), None, 1)
    with pytest.raises(HcpError, match="W must divide 128"):
        ops.conv3x3(pack, x, (1, 64, 96))
    qkv = torch.zeros(1, 16, 3 * 200, dtype=BF, device=DEV)
    with pytest.raises(HcpError, match="head dim"):
        ops.attention(1, 200, (0, 200, 400), qkv)
    a, w = torch.zeros(16, 64, dtype=BF, device=DEV), torch.zeros(12, 64, dtype=BF, device=DEV)
    with pytest.raises(HcpError, match="multiple of 8"):
        ops.gemm_raw([(a, 64, 64)], [(w, 64, 12, 0)], 16, 12, torch.empty(16, 16, dtype=BF, device=DEV), 16)
    torch.cuda.synchronize()
    assert _lib.launch_count == before
