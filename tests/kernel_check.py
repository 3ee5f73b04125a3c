"""Strict comparison of a kernel result with an fp64 reference, and canary buffers that catch stray writes.

The reference is computed in float64 from the bf16-rounded operands the kernel actually reads, so the only differences left are
the kernel's fp32 accumulation order and the bf16 rounding of its output.  Each check reports three numbers and bounds all of them:

  rel     relative L2 over the whole tensor                                        ||got - ref|| / ||ref||
  block   worst relative L2 over the kernel's own tiles (128 rows x BN columns for GEMM / convolution, 64 query rows x one head for
          attention).  One wrong tile among thousands moves `rel` by only sqrt(1/tiles); here it fails on its own.
  maxabs  max |got - ref| / max |ref|: a few wrong elements inside an otherwise right tile.

Any NaN or Inf in a result fails; an output element the kernel never wrote keeps the canary's NaN pattern and fails that way.

Each bound is about 2-3x the worst value measured over every case of tests/test_gpu_edges.py on one H100 80GB HBM3 (400 W power
limit; errors do not depend on it), and tighter than the 1e-2 / 2e-2 relative L2 the per-op tests of tests/test_gpu_parity.py use.
bf16 keeps 8 significand bits, so rounding an output alone costs up to 2^-9 = 2.0e-3 relative per element, ~1.1e-3 in L2:

                                                       measured worst (rel / block / maxabs)    bound
  FWD   GEMM / convolution / attention forward, LoRA   2.97e-3 / 3.02e-3 / 4.25e-3              6e-3 / 8e-3 / 1.2e-2
        linear output and input gradients (one bf16 rounding of an fp32 sum; merged adapters: plus the bf16 merged weight)
  GRAD  attention dQ / dK / dV (P and dS are rounded    2.76e-3 / 4.43e-3 / 5.66e-3              6e-3 / 1e-2 / 1.5e-2
        to bf16 before their MMAs, the result again)
  LORA  LoRA factor gradients (fp32 atomics over       2.50e-3 / 2.59e-3 / 3.19e-3              6e-3 / 8e-3 / 1e-2
        bf16 rank products T / U)
  LSE   attention lse (fp32 natural log; absolute)     1.07e-3                                  3e-3

The normalisation, weight-gradient and time-embedding kernels (tests/test_gpu_norm_wgrad_edges.py, same H100):

  NORM    GroupNorm / LayerNorm y and dx (fp32         1.69e-3 / 2.15e-3 / 3.51e-3              4e-3 / 6e-3 / 9e-3
          statistics, one bf16 rounding of the output)
  STAT    GroupNorm / LayerNorm mean (in units of the  4.3e-8 (mean) / 5.5e-7 (rstd)             1.5e-6
          standard deviation) and rstd (relative), fp32
  F32SUM  fp32 sums of bf16 (or fp32) products: weight  6.00e-7 / 6.09e-7 / 7.27e-7              1.5e-6 / 1.5e-6 / 2e-6
          gradients, column sums, affine gradients, the
          small time-embedding linears, the boundary convolutions' fp32 outputs
  F32SIN  the skinny linear on sinusoidal embeddings    6.05e-6 / 6.83e-6 / 1.01e-5              2e-5 / 2e-5 / 3e-5
          of timesteps up to 999 (fp32 argument t * freq)

The Conv2d LoRA (LoCon) and DreamArtist++ convolution path (tests/test_gpu_lora_conv_edges.py, same H100):

  FWD     the convolution with its LoRA K-segment       1.67e-3 / 1.69e-3 / 3.27e-3
  F32SUM  dW_down (nine shifted-box launches), dW_up,   3.66e-7 / 3.88e-7 / 5.31e-7
          d_rowbias
  LORA    factor gradients end to end (U / T rounded    2.64e-3 / 2.92e-3 / 3.71e-3
          to bf16), against the fp32 masters
  LOCON   y and dX end to end against the fp32 masters  3.06e-3 / 3.10e-3 / 5.21e-3              8e-3 / 8e-3 / 1.2e-2
          (T / U and the factors rounded to bf16 before
          their MMAs), and dX = dgrad(dY, W) accumulated
          in place with dgrad(U, W_down) (two roundings)

The linear LoRA factor gradients (tests/test_gpu_lora_linear_grad.py: hcp_lora_grad_pair and hcp_lora_grad, one H100 80GB HBM3 at
a 700 W power limit).  The error grows linearly with the 128-row tiles one CTA chains in its wgmma accumulator, 1.24e-7 - 1.32e-7
relative per tile in every case above 6 tiles, and it is biased: the results come out smaller in magnitude (the error's projection
on the result is -0.86 of its length, as from adds into the accumulator that round toward zero).  F32SUM was set from chains of at
most 5 tiles (the weight-gradient cases above), so longer chains are bounded by f32sum_chain, F32SUM scaled by the chain over 6:

  F32SUM  dW_down, dW_up, chains of <= 6 tiles          7.27e-7 / 7.43e-7 / 8.91e-7              1.5e-6 / 1.5e-6 / 2e-6
          pair launch against two single launches       8.61e-7 / 8.61e-7 / 1.13e-6
  f32sum_chain(t)  chains of t = 8 - 17 tiles (SD1.5    2.20e-6 / 2.23e-6 / 2.66e-6 at t = 16 / 17  F32SUM x t / 6
          ff proj and SDXL ff at batch 2: 13 / 16)

The training-step and elementwise kernels (tests/test_gpu_step_edges.py, one H100 80GB HBM3 at a 700 W power limit), each error
per element against float64 (worst over all cases and two runs -- the atomics' order varies; bounds are constants of that file):

                                                       measured worst                           bound
  hcp_sumsq (up to 2^28 + 3 squares, relative)         1.66e-6                                  5e-6
  AdamW m', v' / (|beta m| + |(1 - beta) g|)            3.47e-7                                  1e-6
  AdamW p' - 2^-22 |p|, over lr |update| (fp32         5.31e-6                                  1.5e-5
          1 - beta2^step loses digits at small steps)
  EMA / (|e| + |p - e|)                                 1.07e-7                                  3e-7
  add_noise / (sqrt(a) |x0| + sqrt(1 - a) |noise|)      1.30e-7                                  3e-7
  MSE / Min-SNR loss / mean (fixed-order sums)          2.85e-7                                  1e-6
  dpred (relative)                                      4.38e-7                                  1e-6
  CFG mix / (|u| + |s| (|u| + |c|))                     1.55e-7                                  4e-7
  GEGLU, exact GELU, quick-GELU fwd / bwd, in bf16     0.503 (not correctly rounded: at most    1
          ulps of the exact value                       1.6e-4 of the elements)
  dropout with residual and row bias, bf16 ulps        0.500                                    1
          (after the fp32 rounding of the sum)
  hcp_silu_f32 (fp32 output), bf16 ulps                3.5e-3                                   1e-2
  dropout mask, upsample, add, cast, fp32 fan-in sum   bit-exact                                bit-exact
"""
from dataclasses import dataclass

import torch

CANARY = -1          # int16 view of the bf16 bit pattern 0xFFFF (a NaN no kernel produces from finite inputs)


@dataclass(frozen=True)
class Tol:
    rel: float
    block: float
    maxabs: float


FWD = Tol(rel=6e-3, block=8e-3, maxabs=1.2e-2)
GRAD = Tol(rel=6e-3, block=1e-2, maxabs=1.5e-2)
LORA = Tol(rel=6e-3, block=8e-3, maxabs=1e-2)
LSE_ABS = 3e-3
NORM = Tol(rel=4e-3, block=6e-3, maxabs=9e-3)
STAT = 1.5e-6
F32SUM = Tol(rel=1.5e-6, block=1.5e-6, maxabs=2e-6)
F32SIN = Tol(rel=2e-5, block=2e-5, maxabs=3e-5)
LOCON = Tol(rel=8e-3, block=8e-3, maxabs=1.2e-2)


def f32sum_chain(tiles_per_cta: int) -> Tol:
    """F32SUM for a tensor-core weight gradient whose CTAs each chain `tiles_per_cta` 128-row tiles in one wgmma accumulator.  The
    accumulator's error is biased toward smaller magnitudes and grows linearly with the chain (about 1.3e-7 relative per tile), so
    F32SUM, measured on chains of at most 6 tiles, is scaled by the chain beyond that."""
    s = max(1.0, tiles_per_cta / 6)
    return Tol(rel=F32SUM.rel * s, block=F32SUM.block * s, maxabs=F32SUM.maxabs * s)


def compare(name: str, got: torch.Tensor, ref: torch.Tensor, tol: Tol, block=(128, 128)) -> None:
    """got / ref [..., R, C]; blocks of block[0] rows x block[1] columns over the last two dimensions (leading dimensions, e.g.
    images, are separate blocks).  Prints the three errors, then asserts them against `tol`; a failure names the worst block."""
    got = got.detach().to(ref.device, torch.float64)
    ref = ref.detach().to(torch.float64)
    assert got.shape == ref.shape, f"{name}: shape {tuple(got.shape)} != {tuple(ref.shape)}"
    bad = int((~torch.isfinite(got)).sum())
    assert bad == 0, f"{name}: {bad} NaN / Inf elements"
    diff = got - ref
    rel = float(diff.norm() / ref.norm().clamp_min(1e-300))
    maxabs = float(diff.abs().max() / ref.abs().max().clamp_min(1e-300))
    R, Cn = ref.shape[-2], ref.shape[-1]
    br, bc = min(block[0], R), min(block[1], Cn)
    pr, pc = (-R) % br, (-Cn) % bc

    def per_block(t):
        t = torch.nn.functional.pad(t.reshape(-1, R, Cn).square(), (0, pc, 0, pr))
        return t.reshape(t.shape[0], (R + pr) // br, br, (Cn + pc) // bc, bc).sum((2, 4)).sqrt()

    blk = per_block(diff) / per_block(ref).clamp_min(1e-300)
    worst = int(blk.argmax())
    lead, rest = divmod(worst, blk.shape[1] * blk.shape[2])
    where = (lead, (rest // blk.shape[2]) * br, (rest % blk.shape[2]) * bc)
    wb = float(blk.max())
    msg = (f"{name}: rel={rel:.3e} (<= {tol.rel:.1e}), worst block {wb:.3e} (<= {tol.block:.1e}) at lead {where[0]} row {where[1]} "
           f"col {where[2]}, maxabs={maxabs:.3e} (<= {tol.maxabs:.1e})")
    print(msg)
    assert rel <= tol.rel and wb <= tol.block and maxabs <= tol.maxabs, msg


class Canary:
    """A bf16 (or fp32: `dtype=torch.float32`, pattern 0xFFFFFFFF) buffer of `rows + 2 * pad` rows x `ld` columns prefilled with all
    ones; `view` is the rows x cols output rectangle that starts `pad` rows down and `col0` columns in.  `check()` asserts that no
    element outside the rectangle changed, bit for bit."""

    def __init__(self, rows: int, cols: int, ld: int = 0, pad: int = 3, col0: int = 8, device="cuda", dtype=torch.bfloat16):
        ld = ld or (cols + 71) // 8 * 8
        assert col0 + cols <= ld and ld % 8 == 0 and col0 % 8 == 0
        self.bits = torch.int16 if dtype == torch.bfloat16 else torch.int32
        assert dtype in (torch.bfloat16, torch.float32)
        self.buf = torch.full((rows + 2 * pad, ld), CANARY, dtype=self.bits, device=device).view(dtype)
        self.view = self.buf[pad:pad + rows, col0:col0 + cols]
        self.ld, self.rect = ld, (pad, pad + rows, col0, col0 + cols)

    def check(self, name: str) -> None:
        bits = self.buf.view(self.bits).clone()
        r0, r1, c0, c1 = self.rect
        bits[r0:r1, c0:c1] = CANARY
        stray = int((bits != CANARY).sum())
        assert stray == 0, f"{name}: {stray} elements outside the output rectangle were written"
