"""GPU tests of the kernels either side of the UNet call and of the small bf16 / fp32 elementwise kernels, at their edges
(`pytest -m gpu`).

Every kernel is called through its C ABI and compared element by element with a float64 restatement computed from the exact fp32 /
bf16 values it reads:
  * optimizer and clip: hcp_sumsq past its 592-block grid-stride wave, hcp_adamw_flat_dev one step at a time from the kernel's own
    state (tail-only sizes, one wave of 16 blocks per SM exactly / one float4 short / one over, an offset segment of the flat buffer,
    the clip engaged or not, data-parallel grad_scale, hyper-parameters rewritten between steps), hcp_adamw_flat, hcp_ema_flat up to
    the decay_max clamp;
  * losses and noise: hcp_add_noise, hcp_mse_loss and the four hcp_snr_mse_loss weights at both SNR extremes (t = 0 / 999), grid
    strides, accumulation into a non-zero loss, dpred = NULL, grad_scale != 1; hcp_cfg_mix_f32 at t = 0, 1, T-2, T-1;
  * dropout: the keep mask bit for bit against tests/philox_ref.py (Philox4x32-10), column ranges inside wider rows, seeds and draw
    counters with high bits set, the residual / row-bias epilogue, the same mask on the gradient;
  * GEGLU, exact GELU, quick-GELU and SiLU within one bf16 ulp of the exact function over [-12, 12], +-0, tiny values and +-60;
    upsample, add, cast and the fp32 fan-in sum bit-exact;
  * bad sizes and misaligned buffers refused before any launch, empty sizes as no-ops.
Outputs land in canary buffers (bit pattern 0xFFFF / 0xFFFFFFFF) whose surroundings must stay untouched.  Each bound sits at 2-3x
the worst error measured on one H100 80GB HBM3 (tests/kernel_check.py lists both).
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from kernel_check import CANARY, Canary
from philox_ref import dropout_keep

pytestmark = pytest.mark.gpu

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
HCP_ERR_INVALID = -1
GRID_CAP = 592                  # blocks of hcp_sumsq / hcp_mse_loss / hcp_snr_mse_loss; larger sizes take the grid-stride loop

# bounds (errors in the units named; measured worst on the H100 in tests/kernel_check.py)
SUMSQ_REL = 5e-6                # |got - ref| / ref, fp32 partial sums of up to 2^28 squares, 592 of them added with atomics
ADAM_MV = 1e-6                  # m', v': |got - ref| / (|beta m| + |(1 - beta) g|)
ADAM_P = 1.5e-5                   # p': (|got - ref| - 2^-22 |p|) / (lr |m^ / (sqrt v^ + eps)|): relative to the update once the fp32
                                #     roundings of p are allowed for; fp32 1 - beta2^step loses digits at small steps
EMA_REL = 3e-7                  # |got - ref| / (|e| + |p - e|)
NOISE_REL = 3e-7                # |got - ref| / (sqrt(a) |x0| + sqrt(1 - a) |noise|)
LOSS_REL = 2e-5                 # |loss - ref| / mean(w d^2): 592 block partials added with fp32 atomics onto a running total
DPRED_REL = 1e-6                # per element |got - ref| / |ref|
CFG_REL = 4e-7                  # |got - ref| / (|u| + |s| (|u| + |c|)) forward, / ((1 + |s|) |g|) backward
ULP = 1.0                       # the bf16 elementwise kernels: within one bf16 ulp of the exact value
SILU_ULP = 1e-2                 # hcp_silu_f32 (fp32 out), in bf16 ulps: __expf and the cancellation of 1 + z (1 - s) near z = -1.28


def measured(name: str, value: float, bound: float) -> None:
    """Print one measured error next to its bound (the lines kernel_check.py's table is made from), then assert it."""
    print(f"MEASURED {name}: {value:.3e} (<= {bound:.1e})")
    assert value <= bound, f"{name}: {value:.3e} > {bound:.1e}"


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(seed: int) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(seed)


class FlatCanary:
    """fp32 (or bf16) [lo + n + 8] prefilled with all ones bits; `view` = elements [lo, lo + n).  `check()` asserts that no element
    outside the view changed."""

    def __init__(self, n: int, lo: int = 8, values=None, dtype=F32):
        self.bits = torch.int32 if dtype == F32 else torch.int16
        self.buf = torch.full((lo + n + 8,), -1, dtype=self.bits, device=DEV).view(dtype)
        self.view = self.buf[lo:lo + n]
        if values is not None:
            self.view.copy_(values)
        self.lo, self.n = lo, n

    def check(self, name: str) -> None:
        b = self.buf.view(self.bits)
        stray = int((b[:self.lo] != -1).sum()) + int((b[self.lo + self.n:] != -1).sum())
        assert stray == 0, f"{name}: {stray} elements outside [lo, lo + n) were written"


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 at |x| (float64): 2^(e - 7) for |x| in [2^e, 2^(e+1)), 2^-133 below the smallest normal."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def ulps(name: str, got: torch.Tensor, ref: torch.Tensor, bound: float = ULP) -> None:
    """Every element of `got` within `bound` bf16 ulps of the exact float64 `ref`; prints the worst and the share not equal to
    ref rounded once."""
    g = got.double()
    assert bool(torch.isfinite(g).all()), f"{name}: {int((~torch.isfinite(g)).sum())} NaN / Inf elements"
    err = ((g - ref).abs() / bf16_ulp(ref)).max()
    inexact = float((got != ref.to(got.dtype) if got.dtype == BF else got.to(BF) != ref.to(BF)).double().mean())
    print(f"{name}: {inexact:.2e} of the elements not the correctly rounded value")
    measured(f"{name} ulps", float(err), bound)


# ----------------------------------------------------------------------------------------------------------------------------------
# optimizer and clip
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 255, 256, 257, GRID_CAP * 256 + 1, 2 ** 24 + 5, 2 ** 28 + 3])
def test_sumsq_grid_stride_and_accumulation(n):
    """out += sum g^2 from a non-zero start; sizes past 592 x 256 take the grid-stride loop (2^28 + 3 fp32 is 1 GB).  The last
    element is large, so that losing it alone (592 x 256 + 1) fails."""
    g = torch.randn(n, generator=gen(n % 1000), device=DEV)
    g[-1] = 8.0
    s = sum(float(g[i:i + 2 ** 26].double().square().sum()) for i in range(0, n, 2 ** 26))
    out = torch.full((1,), 0.75 * s, device=DEV)                  # a start of the sum's size: its own rounding stays below the bound
    start = float(out)
    call("hcp_sumsq", g.data_ptr(), n, out.data_ptr(), stream_ptr())
    measured(f"sumsq n={n} rel", abs(float(out) - start - s) / s, SUMSQ_REL)


def adamw_ref(p, g, m, v, hyper, step, gscale, sumsq, max_norm):
    """torch.optim.AdamW (decoupled decay, bias corrections at the post-increment step) after clip_grad_norm_ on g * gscale, in
    float64 from the fp32 values the kernel reads.  Returns p', m', v' and the scale each error is measured in: for p' the size of
    the update lr |m^ / (sqrt v^ + eps)|, after an allowance of 2^-22 |p| for the fp32 roundings of p (x (1 - lr wd), - update)."""
    lr, b1, b2, eps, wd = (float(h) for h in hyper)
    clip = 1.0
    if sumsq is not None and max_norm > 0:
        clip = min(1.0, max_norm / (math.sqrt(sumsq) * gscale + 1e-6))
    grad = g.double() * gscale * clip
    m0, v0, p0 = m.double(), v.double(), p.double()
    m1 = b1 * m0 + (1 - b1) * grad
    v1 = b2 * v0 + (1 - b2) * grad * grad
    upd = (m1 / (1 - b1 ** step)) / (torch.sqrt(v1 / (1 - b2 ** step)) + eps)
    p1 = p0 * (1 - lr * wd) - lr * upd
    scales = (lr * upd.abs(), (b1 * m0).abs() + ((1 - b1) * grad).abs(), b2 * v0 + (1 - b2) * grad * grad)
    allow = (2.0 ** -22 * p0.abs(), 0.0, 0.0)
    return (p1, m1, v1), scales, allow


# the four steps every size runs: (hyper = lr, beta1, beta2, eps, weight_decay), grad_scale, clip (None: max_norm = 0;
# otherwise max_norm = clip * ||g * grad_scale||: < 1 engages it)
ADAM_STEPS = [((1e-3, 0.9, 0.999, 1e-8, 1e-2), 0.5, 0.3),
              ((5e-4, 0.85, 0.999, 1e-8, 0.0), 1.0, 3.0),            # beta1 rewritten between calls, as OneCycleLR does
              ((2e-3, 0.95, 0.99, 1e-6, 1e-2), 0.5, None),
              ((1e-3, 0.9, 0.98, 1e-8, 0.0), 1.0, 0.5)]


# (n, lo): n < 0 stands for 4 (cap4 + d) + r with d = -n // 4 - 2 and r = -n % 4, cap4 = 256 x 16 x SMs float4 (one grid-stride wave
# of hcp_adamw_flat_dev; the SM count is only known on the device)
ADAM_SIZES = [(n, 8) for n in (1, 2, 3, 4, 5)] + [(-(4 * (d + 2) + r), 8) for d in (-1, 0, 1) for r in (0, 1, 3)]
ADAM_SIZES.append((1000003, 36))                               # a segment at flat + 4 lo, lo % 4 == 0 and lo % 256 != 0


def adam_n(n: int) -> int:
    if n > 0:
        return n
    d, r = -n // 4 - 2, -n % 4
    return 4 * (256 * 16 * sms() + d) + r


def run_adam(n, lo, dev_hyper: bool, seed=0):
    g = gen(seed)
    p = FlatCanary(n, lo, torch.randn(n, generator=g, device=DEV))
    m = FlatCanary(n, lo, 0.1 * torch.randn(n, generator=g, device=DEV))
    v = FlatCanary(n, lo, 0.01 * torch.randn(n, generator=g, device=DEV).square())
    grad = FlatCanary(n, lo)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    hyper = torch.zeros(5, device=DEV)
    sumsq = torch.zeros(1, device=DEV)
    worst = [0.0, 0.0, 0.0]
    for k, (hy, gscale, clip) in enumerate(ADAM_STEPS, start=1):
        grad.view.copy_(torch.randn(n, generator=g, device=DEV) * (1 + k))
        hyper.copy_(torch.tensor(hy))
        sumsq.fill_(float(grad.view.double().square().sum()))
        ss = float(sumsq)
        max_norm = 0.0 if clip is None else clip * math.sqrt(ss) * gscale
        before = [t.view.clone() for t in (p, m, v)]
        hyper32 = [float(h) for h in hyper.cpu()]
        if dev_hyper:
            call("hcp_adamw_flat_dev", p.view.data_ptr(), grad.view.data_ptr(), m.view.data_ptr(), v.view.data_ptr(), n, hyper.data_ptr(),
                 gscale, sumsq.data_ptr(), max_norm, step.data_ptr(), stream_ptr())
        else:
            lr = hyper[0:1]
            call("hcp_adamw_flat", p.view.data_ptr(), grad.view.data_ptr(), m.view.data_ptr(), v.view.data_ptr(), n, lr.data_ptr(),
                 hyper32[1], hyper32[2], hyper32[3], hyper32[4], gscale, sumsq.data_ptr(), max_norm, step.data_ptr(), stream_ptr())
        assert int(step) == k
        ss32 = float(np.float32(ss))
        refs, scales, allow = adamw_ref(before[0], grad.view, before[1], before[2], hyper32, k, gscale, ss32, float(np.float32(max_norm)))
        for j, (t, r, s, a) in enumerate(zip((p, m, v), refs, scales, allow)):
            e = float((((t.view.double() - r).abs() - a).clamp_min(0) / s.clamp_min(1e-30)).max())
            worst[j] = max(worst[j], e)
    for t, name in zip((p, m, v, grad), "pmvg"):
        t.check(f"adamw n={n} {name}")
    return worst


@pytest.mark.parametrize("n,lo", ADAM_SIZES)
def test_adamw_flat_dev_per_step(n, lo):
    """hcp_adamw_flat_dev four steps from its own state, each step against the float64 restatement: tail-only sizes (n < 4), the
    grid cap 256 x 16 x SMs float4 exactly / -1 / +1 with n % 4 in {0, 1, 3}, and an offset segment of the flat buffer."""
    n = adam_n(n)
    wp, wm, wv = run_adam(n, lo, dev_hyper=True)
    measured(f"adamw_dev n={n} lo={lo} m", wm, ADAM_MV)
    measured(f"adamw_dev n={n} lo={lo} v", wv, ADAM_MV)
    measured(f"adamw_dev n={n} lo={lo} p", wp, ADAM_P)


@pytest.mark.parametrize("n", [1, 5, 257, 70001])
def test_adamw_flat_host_scalars(n):
    """hcp_adamw_flat (betas, eps and weight decay as host scalars, lr on the device): the same restatement."""
    wp, wm, wv = run_adam(n, 8, dev_hyper=False, seed=1)
    measured(f"adamw n={n} m", wm, ADAM_MV)
    measured(f"adamw n={n} v", wv, ADAM_MV)
    measured(f"adamw n={n} p", wp, ADAM_P)


@pytest.mark.parametrize("decay_max,inv_gamma,power", [(0.9997, 1.0, 2 / 3), (0.999, 7.5, 0.75)])
def test_ema_flat_steps_and_clamp(decay_max, inv_gamma, power):
    """ema = lerp(ema, p, 1 - decay), decay = clip(1 - (1 + step / inv_gamma)^-power, 0, decay_max), at steps 1 .. 10^7 (the last
    clamped by decay_max) and sizes with 256-thread tails."""
    dm, ig, pw = (float(np.float32(x)) for x in (decay_max, inv_gamma, power))
    for n in (1, 255, 257, 65537):
        for step_v in (1, 2, 10, 10 ** 4, 10 ** 7):
            g = gen(n + step_v)
            e = FlatCanary(n, 8, torch.randn(n, generator=g, device=DEV))
            p = torch.randn(n, generator=g, device=DEV)
            e0 = e.view.double().clone()
            step = torch.full((1,), step_v, dtype=torch.int32, device=DEV)
            call("hcp_ema_flat", e.view.data_ptr(), p.data_ptr(), n, step.data_ptr(), decay_max, inv_gamma, power, stream_ptr())
            decay = min(max(1 - (1 + step_v / ig) ** -pw, 0.0), dm)
            ref = e0 + (1 - decay) * (p.double() - e0)
            err = float(((e.view.double() - ref).abs() / (e0.abs() + (p.double() - e0).abs())).max())
            measured(f"ema n={n} step={step_v} decay_max={decay_max}", err, EMA_REL)
            e.check(f"ema n={n} step={step_v}")


# ----------------------------------------------------------------------------------------------------------------------------------
# losses and noise
# ----------------------------------------------------------------------------------------------------------------------------------
T_CYCLE = [0, 999, 500, 1, 998]


def acp_dev():
    return U.ddpm_alphas_cumprod().to(DEV)


@pytest.mark.parametrize("B,per_image", [(1, 1), (1, 252), (5, 572), (16, 572), (16, 4 * 64 * 64)])
def test_add_noise_edges(B, per_image):
    """x_t = sqrt(acp[t]) x0 + sqrt(1 - acp[t]) noise at t in {0, 1, 500, 998, 999}, images not a multiple of 256 elements."""
    acp = acp_dev()
    g = gen(B * per_image)
    x0 = torch.randn(B * per_image, generator=g, device=DEV)
    noise = torch.randn(B * per_image, generator=g, device=DEV)
    t = torch.tensor([T_CYCLE[b % 5] for b in range(B)], dtype=torch.int64, device=DEV)
    xt = FlatCanary(B * per_image)
    call("hcp_add_noise", x0.data_ptr(), noise.data_ptr(), t.data_ptr(), acp.data_ptr(), B, per_image, xt.view.data_ptr(), stream_ptr())
    a = acp.double()[t].repeat_interleave(per_image)
    sa, sb = a.sqrt(), (1 - a).sqrt()
    ref = sa * x0.double() + sb * noise.double()
    err = float(((xt.view.double() - ref).abs() / (sa * x0.double().abs() + sb * noise.double().abs())).max())
    measured(f"add_noise B={B} per_image={per_image}", err, NOISE_REL)
    xt.check("add_noise")


def snr_weight(a: torch.Tensor, gamma: float, mode: int) -> torch.Tensor:
    """min_snr_loss.py's four weights in float64 (a = acp[t] as fp32 read by the kernel); mode -1 = plain MSE."""
    if mode < 0:
        return torch.ones_like(a)
    snr = a / (1 - a)
    if mode == 0:
        return torch.clamp(gamma / snr, max=1.0)
    if mode == 1:
        return gamma ** 3 / (snr ** 2 + gamma ** 3)
    if mode == 2:
        return 4 * (gamma * snr) ** 2 / (snr ** 2 + gamma ** 2) ** 2
    s2 = 1 - a
    return (s2 + gamma ** 2) / (snr * s2 * gamma ** 2)


@pytest.mark.parametrize("B,per_image", [(1, 1), (3, 1), (5, 51), (1, 257), (7, 21651), (5, 3355445)])
def test_mse_and_snr_losses(B, per_image):
    """hcp_mse_loss and hcp_snr_mse_loss (modes 0-3, gamma 1 and 5) with t at both SNR extremes: loss accumulated into a non-zero
    start, dpred
    per element with grad_scale 0.5, and the same loss again with dpred = NULL.  7 x 21651 and 5 x 3355445 take the grid stride."""
    acp = acp_dev()
    n = B * per_image
    g = gen(n)
    pred = torch.randn(n, generator=g, device=DEV)
    target = torch.randn(n, generator=g, device=DEV)
    t = torch.tensor([T_CYCLE[b % 5] for b in range(B)], dtype=torch.int64, device=DEV)
    d = pred.double() - target.double()
    a = acp.double()[t]
    for mode, gamma in [(-1, 1.0)] + [(m, gm) for m in range(4) for gm in (1.0, 5.0)]:
        w = snr_weight(a, gamma, mode).repeat_interleave(per_image)
        mean = float((w * d * d).sum()) / n
        ref_d = 2 * w * d * 0.5 / n
        loss = torch.full((1,), 0.75 * mean, device=DEV)           # accumulate (+=) onto a start of the mean's size
        start = float(loss)
        loss_nodp = torch.zeros(1, device=DEV)
        dpred = FlatCanary(n)
        for l_, dp in ((loss, dpred.view.data_ptr()), (loss_nodp, None)):
            if mode < 0:
                call("hcp_mse_loss", pred.data_ptr(), target.data_ptr(), n, 0.5, l_.data_ptr(), dp, stream_ptr())
            else:
                call("hcp_snr_mse_loss", pred.data_ptr(), target.data_ptr(), t.data_ptr(), acp.data_ptr(), gamma, mode, per_image, n, 0.5,
                     l_.data_ptr(), dp, stream_ptr())
        tag = f"loss mode={mode} gamma={gamma} n={n}"
        measured(f"{tag} loss", abs(float(loss) - start - mean) / mean, LOSS_REL)
        measured(f"{tag} loss (dpred NULL)", abs(float(loss_nodp) - mean) / mean, LOSS_REL)
        err = float(((dpred.view.double() - ref_d).abs() / ref_d.abs().clamp_min(1e-38)).max())
        measured(f"{tag} dpred", err, DPRED_REL)
        dpred.check(tag)


@pytest.mark.parametrize("mode,lo,hi", [(0, 1.5, 4.0), (1, 1.5, 4.0), (2, 1.5, 4.0), (1, 2.5, 2.5)])
def test_cfg_mix_edges(mode, lo, hi):
    """DreamArtist CFG mix forward and backward at t = 0, 1, T-2, T-1 for the three rate shapes and the constant scale, images of
    572 elements (not a multiple of 256)."""
    T, B, per = 1000, 4, 572
    t = torch.tensor([0, 1, T - 2, T - 1], dtype=torch.int64, device=DEV)
    g = gen(mode)
    eps2 = torch.randn(2 * B * per, generator=g, device=DEV)
    dout = torch.randn(B * per, generator=g, device=DEV)
    lo32, hi32 = float(np.float32(lo)), float(np.float32(hi))
    rate = t.double() / (T - 1)
    if mode == 1:
        rate = torch.cos((rate - 1) * math.pi / 2)
    elif mode == 2:
        rate = 1 - torch.cos(rate * math.pi / 2)
    s = (torch.full_like(rate, lo32) if lo == hi else (hi32 - lo32) * rate + lo32).repeat_interleave(per)
    u, c = eps2[:B * per].double(), eps2[B * per:].double()
    out = FlatCanary(B * per)
    call("hcp_cfg_mix_f32", eps2.data_ptr(), None, t.data_ptr(), B, per, lo, hi, mode, T, out.view.data_ptr(), stream_ptr())
    ref = u + s * (c - u)
    measured(f"cfg fwd mode={mode} lo={lo} hi={hi}", float(((out.view.double() - ref).abs() / (u.abs() + s.abs() * (u.abs() + c.abs()))).max()),
             CFG_REL)
    out.check("cfg fwd")
    d2 = FlatCanary(2 * B * per)
    call("hcp_cfg_mix_f32", None, dout.data_ptr(), t.data_ptr(), B, per, lo, hi, mode, T, d2.view.data_ptr(), stream_ptr())
    gd = dout.double()
    ref2 = torch.cat([(1 - s) * gd, s * gd])
    scale2 = torch.cat([(1 + s.abs()) * gd.abs()] * 2)
    measured(f"cfg bwd mode={mode} lo={lo} hi={hi}", float(((d2.view.double() - ref2).abs() / scale2).max()), CFG_REL)
    d2.check("cfg bwd")


# ----------------------------------------------------------------------------------------------------------------------------------
# dropout: the mask restated bit for bit
# ----------------------------------------------------------------------------------------------------------------------------------
def dropout_state(seed: int, draw: int) -> torch.Tensor:
    return torch.from_numpy(np.array([seed, draw], dtype=np.uint64).view(np.int64)).to(DEV)


def bounded_x(rows, ld, seed):
    """bf16 [rows, ld] with |x| in [0.5, 1.5): an output of 0 can only mean the element was dropped."""
    g = gen(seed)
    mag = 0.5 + torch.rand(rows, ld, generator=g, device=DEV)
    sign = torch.where(torch.rand(rows, ld, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    return (mag * sign).to(BF)


# rows, ncols, ldx, c0 (first column of the range), p, seed, draw advance past 2^32
DROP_CASES = [
    (16, 64, 64, 0, 0.0, 1, False),
    (37, 136, 200, 16, 0.1, 0x5DEECE66D1234567, False),        # range inside a wider row, 629 vectors (not a multiple of 256)
    (37, 136, 200, 48, 0.5, 0x5DEECE66D1234567, True),         # draw counter >= 2^32: draw_hi enters the key
    (301, 512, 512, 0, 0.999, 0x0123456789ABCDEF, True),
]


@pytest.mark.parametrize("rows,ncols,ldx,c0,p,seed,adv", DROP_CASES)
def test_dropout_mask_bit_exact(rows, ncols, ldx, c0, p, seed, adv):
    """The keep mask equals tests/philox_ref.py's restatement bit for bit, kept values are bf16(x * (1 / (1 - p))) exactly, nothing
    outside the column range or the rows is written, and the gradient call with the same (state, site) applies the same mask."""
    site = 7
    state = dropout_state(seed, 5)
    if adv:
        call("hcp_counter_add_u64", state.data_ptr() + 8, 1 << 32, stream_ptr())
    draw = int(state.cpu().numpy().view(np.uint64)[1])
    assert draw == (5 + (1 << 32) if adv else 5)
    keep = torch.from_numpy(dropout_keep(rows, ncols, p, seed, draw, site)).to(DEV)
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    for what, x_seed in (("forward", 11), ("gradient", 12)):
        x = bounded_x(rows, ldx, x_seed)
        out = Canary(rows, ncols, ld=ldx + 64, col0=c0 + 8)
        call("hcp_dropout_bf16", x.data_ptr() + 2 * c0, ldx, None, 0, None, 0, 1, rows, ncols, p, state.data_ptr(), site,
             out.view.data_ptr(), out.ld, stream_ptr())
        got = out.view
        xs = x[:, c0:c0 + ncols]
        mism = int(((got != 0) != keep).sum())
        assert mism == 0, f"dropout {what} p={p}: {mism} of {keep.numel()} mask bits differ from the Philox restatement"
        want = torch.where(keep, (xs.float() * inv).to(BF), torch.zeros_like(xs))
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"dropout {what} p={p}: kept values not bf16(x / (1 - p))"
        out.check(f"dropout {what} p={p}")
    print(f"dropout p={p}: kept {float(keep.double().mean()):.4f}")


def test_dropout_residual_rowbias_epilogue():
    """out = keep x / (1 - p) + residual + rowbias[r / HW] (rows_per_group = HW, rowbias_ld != ncols) within one bf16 ulp of the
    float64 value on the restated mask (plus the fp32 rounding of the three-term sum, which FMA contraction may reorder)."""
    B, HW, ncols, ldx, c0, p = 3, 37, 136, 200, 16, 0.25
    rows = B * HW
    seed, site = 0x7FEDCBA987654321, 3
    state = dropout_state(seed, 9)
    call("hcp_counter_add_u64", state.data_ptr() + 8, 1 << 32, stream_ptr())
    keep = torch.from_numpy(dropout_keep(rows, ncols, p, seed, 9 + (1 << 32), site)).to(DEV)
    x = bounded_x(rows, ldx, 21)
    res = (torch.randn(rows, ldx, generator=gen(22), device=DEV)).to(BF)
    rb_ld = 160
    rowbias = torch.randn(B, rb_ld, generator=gen(23), device=DEV)
    out = Canary(rows, ncols, ld=ldx + 64, col0=c0 + 8)
    call("hcp_dropout_bf16", x.data_ptr() + 2 * c0, ldx, res.data_ptr() + 2 * c0, ldx, rowbias.data_ptr() + 4 * c0, rb_ld, HW, rows, ncols,
         p, state.data_ptr(), site, out.view.data_ptr(), out.ld, stream_ptr())
    inv = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    xd = torch.where(keep, x[:, c0:c0 + ncols].double() * inv, torch.zeros_like(keep, dtype=F64))
    rd = res[:, c0:c0 + ncols].double()
    bd = rowbias[:, c0:c0 + ncols].double().repeat_interleave(HW, 0)
    ref = xd + rd + bd
    slack = 2.0 ** -22 * (xd.abs() + rd.abs() + bd.abs())            # fp32 rounding of the sum before the bf16 rounding
    err = float(((out.view.double() - ref).abs() / (bf16_ulp(ref) + slack)).max())
    measured("dropout epilogue ulps", err, ULP)
    out.check("dropout epilogue")


# ----------------------------------------------------------------------------------------------------------------------------------
# bf16 / fp32 elementwise kernels
# ----------------------------------------------------------------------------------------------------------------------------------
SPECIAL = [0.0, -0.0, 1e-30, -1e-30, 1.2e-38, -1.2e-38, 1e-39, -1e-39, 60.0, -60.0, 12.0, -12.0]


def act_inputs(M, F, seed):
    """bf16 [M, F]: a dense grid over [-12, 12] plus +-0, tiny normals and subnormals and +-60, in random order."""
    n = M * F
    grid = torch.linspace(-12, 12, max(n - len(SPECIAL), 1), dtype=F64)
    vals = torch.cat([grid, torch.tensor(SPECIAL, dtype=F64)])[:n]
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed))
    return vals[perm].to(BF).reshape(M, F).to(DEV)


def phi_cdf(x):
    return 0.5 * torch.special.erfc(-x / math.sqrt(2))


def gelu64(x):
    return x * phi_cdf(x)


def gelu_grad64(x):
    return phi_cdf(x) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def qgelu64(x):
    return x * torch.sigmoid(1.702 * x)


def qgelu_grad64(x):
    s = torch.sigmoid(1.702 * x)
    return s + 1.702 * x * s * (1 - s)


ACT_SHAPES = [(2309, 8), (231, 3072), (231, 5120)]             # M * F / 8 not a multiple of 256


@pytest.mark.parametrize("M,F", ACT_SHAPES)
def test_geglu_within_one_ulp(M, F):
    """h = a * gelu(g) and du = [dh gelu(g) | dh a gelu'(g)], g over the activation grid."""
    g_ = act_inputs(M, F, 1)
    a = torch.randn(M, F, generator=gen(2), device=DEV).to(BF)
    u = torch.cat([a, g_], 1).contiguous()
    dh = torch.randn(M, F, generator=gen(3), device=DEV).to(BF)
    h = FlatCanary(M * F, dtype=BF)
    call("hcp_geglu_fwd_bf16", u.data_ptr(), M, F, h.view.data_ptr(), stream_ptr())
    ulps(f"geglu fwd M={M} F={F}", h.view.reshape(M, F), a.double() * gelu64(g_.double()))
    h.check("geglu fwd")
    du = FlatCanary(M * 2 * F, dtype=BF)
    call("hcp_geglu_bwd_bf16", u.data_ptr(), dh.data_ptr(), M, F, du.view.data_ptr(), stream_ptr())
    d2 = du.view.reshape(M, 2 * F)
    ulps(f"geglu bwd da M={M} F={F}", d2[:, :F], dh.double() * gelu64(g_.double()))
    ulps(f"geglu bwd dg M={M} F={F}", d2[:, F:], dh.double() * a.double() * gelu_grad64(g_.double()))
    du.check("geglu bwd")


@pytest.mark.parametrize("kind", ["gelu", "quick_gelu"])
@pytest.mark.parametrize("M,F", ACT_SHAPES)
def test_gelu_family_within_one_ulp(kind, M, F):
    """Exact GELU (erfc-based) and quick-GELU forward and backward; at +-60 quick-GELU's __expf overflows and the result must
    stay finite."""
    f, fg = (gelu64, gelu_grad64) if kind == "gelu" else (qgelu64, qgelu_grad64)
    x = act_inputs(M, F, 4)
    dy = torch.randn(M, F, generator=gen(5), device=DEV).to(BF)
    y = FlatCanary(M * F, dtype=BF)
    call(f"hcp_{kind}_fwd_bf16", x.data_ptr(), M, F, y.view.data_ptr(), stream_ptr())
    ulps(f"{kind} fwd M={M} F={F}", y.view.reshape(M, F), f(x.double()))
    y.check(f"{kind} fwd")
    dx = FlatCanary(M * F, dtype=BF)
    call(f"hcp_{kind}_bwd_bf16", x.data_ptr(), dy.data_ptr(), M, F, dx.view.data_ptr(), stream_ptr())
    ulps(f"{kind} bwd M={M} F={F}", dx.view.reshape(M, F), dy.double() * fg(x.double()))
    dx.check(f"{kind} bwd")


def test_silu_f32_within_one_ulp():
    """hcp_silu_f32 (fp32 in and out: the time-embedding path) on the same bf16 grid, forward and dy * silu'."""
    x = act_inputs(1, 70001, 6).float().reshape(-1)
    dy = torch.randn(x.numel(), generator=gen(7), device=DEV)
    for what, dptr, ref in (("fwd", None, x.double() * torch.sigmoid(x.double())),
                            ("bwd", dy.data_ptr(), dy.double() * (torch.sigmoid(x.double()) * (1 + x.double() * (1 - torch.sigmoid(x.double())))))):
        out = FlatCanary(x.numel())
        call("hcp_silu_f32", x.data_ptr(), dptr, x.numel(), out.view.data_ptr(), stream_ptr())
        ulps(f"silu {what}", out.view, ref, SILU_ULP)
        out.check(f"silu {what}")


@pytest.mark.parametrize("H,W,C", [(1, 1, 8), (3, 5, 8), (5, 3, 8), (1, 5, 1280), (3, 3, 1280), (5, 1, 1280)])
def test_upsample2x_bit_exact(H, W, C):
    """Forward: a copy, bit-exact.  Backward: the fp32 sum of each 2x2 block in the kernel's order (dh, then dw), rounded once."""
    B = 2
    x = torch.randn(B, H, W, C, generator=gen(H * W), device=DEV).to(BF)
    y = FlatCanary(B * 4 * H * W * C, dtype=BF)
    call("hcp_upsample2x_fwd_bf16", x.data_ptr(), B, H, W, C, y.view.data_ptr(), stream_ptr())
    want = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(y.view.view(torch.int16), want.reshape(-1).view(torch.int16)), f"upsample fwd {H}x{W}x{C}"
    y.check("upsample fwd")
    dy = (torch.randn(B, 2 * H, 2 * W, C, generator=gen(7), device=DEV) * torch.exp2(torch.randint(-8, 8, (B, 2 * H, 2 * W, C), generator=gen(8),
                                                                                                     device=DEV).float())).to(BF)
    dx = FlatCanary(B * H * W * C, dtype=BF)
    call("hcp_upsample2x_bwd_bf16", dy.data_ptr(), B, H, W, C, dx.view.data_ptr(), stream_ptr())
    blk = dy.float().reshape(B, H, 2, W, 2, C)
    acc = torch.zeros(B, H, W, C, device=DEV)
    for dh in range(2):
        for dw in range(2):
            acc = acc + blk[:, :, dh, :, dw]
    assert torch.equal(dx.view.view(torch.int16), acc.to(BF).reshape(-1).view(torch.int16)), f"upsample bwd {H}x{W}x{C}"
    dx.check("upsample bwd")


@pytest.mark.parametrize("n", [8, 8 * 255, 8 * (256 * 3 + 5)])
def test_add_bf16_bit_exact(n):
    a = torch.randn(n, generator=gen(1), device=DEV).to(BF)
    b = (torch.randn(n, generator=gen(2), device=DEV) * 100).to(BF)
    out = FlatCanary(n, dtype=BF)
    call("hcp_add_bf16", a.data_ptr(), b.data_ptr(), n, out.view.data_ptr(), stream_ptr())
    assert torch.equal(out.view.view(torch.int16), (a.float() + b.float()).to(BF).view(torch.int16))
    out.check("add_bf16")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 1023, 77 * 2048 + 3])
@pytest.mark.parametrize("src_off,dst_off", [(0, 0), (1, 0), (0, 1)])
def test_cast_f32_to_bf16_bit_exact(n, src_off, dst_off):
    """Against .to(torch.bfloat16), NaN and +-inf included, with a canary after n; the source 4 bytes past 16-byte alignment or
    the destination 2 bytes past it takes the element-wise path and gives the same bits."""
    x = torch.randn(n + 4, generator=gen(n), device=DEV) * 1e3
    if n > 1:
        x[1 + src_off] = float("nan")
    if n > 3:
        x[2 + src_off], x[3 + src_off] = float("inf"), float("-inf")
    xs = x[src_off:src_off + n]
    assert (xs.data_ptr() % 16 != 0) == bool(src_off)
    y = FlatCanary(n, lo=8 + dst_off, dtype=BF)
    call("hcp_cast_f32_to_bf16", xs.data_ptr(), n, y.view.data_ptr(), stream_ptr())
    want = xs.to(BF)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(y.view), nan)
    assert bool((y.view[nan].view(torch.int16) != CANARY).all()), "a NaN element was never written"   # NaN bits differ by converter
    assert torch.equal(y.view[~nan].view(torch.int16), want[~nan].view(torch.int16)), f"cast n={n}"
    y.check(f"cast n={n}")


@pytest.mark.parametrize("nsrc", [1, 2, 31, 32, 33, 64, 65, 140])
def test_sum_bf16_to_f32_bit_exact(nsrc):
    """The fp32 fan-in sum equals a sequential fp32 sum in source order, bit for bit; more than 32 sources take several launches
    that accumulate into the output."""
    n = 8 * (256 * 5 + 3)
    g = gen(nsrc)
    srcs = [(torch.randn(n, generator=g, device=DEV) * torch.exp2(torch.randint(-12, 12, (n,), generator=g, device=DEV).float())).to(BF)
            for _ in range(nsrc)]
    out = FlatCanary(n)
    arr = (C.c_void_p * nsrc)(*[s.data_ptr() for s in srcs])
    call("hcp_sum_bf16_to_f32", arr, nsrc, n, out.view.data_ptr(), stream_ptr())
    acc = torch.zeros(n, device=DEV)
    for s in srcs:
        acc = acc + s.float()
    assert torch.equal(out.view.view(torch.int32), acc.view(torch.int32)), f"sum of {nsrc} sources"
    out.check(f"sum nsrc={nsrc}")


# ----------------------------------------------------------------------------------------------------------------------------------
# refusals and empty sizes
# ----------------------------------------------------------------------------------------------------------------------------------
def rc_of(name, *args):
    rc = getattr(_lib.lib(), name)(*args)
    torch.cuda.synchronize()
    return rc


def test_adamw_dev_refusal_leaves_step_counter():
    """A misaligned buffer is refused before the step counter is advanced: a refused call must not move the bias correction of
    every later step."""
    buf = torch.zeros(4, 64, device=DEV)              # p, g, m, v rows of 256 bytes
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0], device=DEV)
    step = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    before = _lib.launch_count
    for k, off in enumerate((4, 8, 12, 4)):               # one of the four buffers off 16-byte alignment
        p, g, m, v = (buf[j].data_ptr() + (off if j == k else 0) for j in range(4))
        rc = rc_of("hcp_adamw_flat_dev", p, g, m, v, 8, hyper.data_ptr(), 1.0, None, 0.0, step.data_ptr(), stream_ptr())
        assert rc == HCP_ERR_INVALID, (k, off)
    assert _lib.launch_count == before
    assert int(step) == 3


def test_negative_sizes_refused_before_launch():
    f = torch.zeros(4096, device=DEV)
    b = torch.zeros(4096, dtype=BF, device=DEV)
    t = torch.zeros(4, dtype=torch.int64, device=DEV)
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0], device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    F_, B_, S = f.data_ptr(), b.data_ptr(), stream_ptr()
    srcs = (C.c_void_p * 1)(B_)
    before = _lib.launch_count
    cases = {
        "hcp_adamw_flat_dev": (F_, F_ + 4096, F_ + 8192, F_ + 12288, -1, hyper.data_ptr(), 1.0, None, 0.0, step.data_ptr(), S),
        "hcp_adamw_flat": (F_, F_ + 4096, F_ + 8192, F_ + 12288, -1, hyper.data_ptr(), 0.9, 0.999, 1e-8, 0.0, 1.0, None, 0.0, step.data_ptr(), S),
        "hcp_sumsq": (F_, -1, F_ + 64, S),
        "hcp_mse_loss": (F_, F_, -1, 1.0, F_ + 64, None, S),
        "hcp_add_noise": (F_, F_, t.data_ptr(), F_, -1, 4, F_ + 64, S),
        "hcp_cast_f32_to_bf16": (F_, -1, B_, S),
        "hcp_geglu_fwd_bf16": (B_, -2, 8, B_ + 1024, S),
        "hcp_geglu_bwd_bf16": (B_, B_, 2, -8, B_ + 1024, S),
        "hcp_gelu_fwd_bf16": (B_, 2, -8, B_ + 1024, S),
        "hcp_gelu_bwd_bf16": (B_, B_, -2, 8, B_ + 1024, S),
        "hcp_quick_gelu_fwd_bf16": (B_, 2, -8, B_ + 1024, S),
        "hcp_quick_gelu_bwd_bf16": (B_, B_, -2, 8, B_ + 1024, S),
        "hcp_upsample2x_fwd_bf16": (B_, -1, 2, 2, 8, B_ + 1024, S),
        "hcp_upsample2x_bwd_bf16": (B_, 1, 2, -2, 8, B_ + 1024, S),
        "hcp_add_bf16": (B_, B_, -8, B_ + 1024, S),
        "hcp_sum_bf16_to_f32": (srcs, 1, -8, F_, S),
    }
    for name, args in cases.items():
        assert rc_of(name, *args) == HCP_ERR_INVALID, name
    assert _lib.launch_count == before
    assert int(step) == 0


def test_empty_sizes_are_noops():
    """n == 0 returns HCP_OK and launches nothing (it used to be a CUDA launch-configuration error for some entry points)."""
    f = torch.full((4096,), 1.5, device=DEV)
    b = torch.zeros(4096, dtype=BF, device=DEV)
    t = torch.zeros(4, dtype=torch.int64, device=DEV)
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0], device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    F_, B_, S = f.data_ptr(), b.data_ptr(), stream_ptr()
    srcs = (C.c_void_p * 2)(B_, B_ + 1024)
    before = _lib.launch_count
    cases = {
        "hcp_adamw_flat_dev": (F_, F_ + 4096, F_ + 8192, F_ + 12288, 0, hyper.data_ptr(), 1.0, None, 0.0, step.data_ptr(), S),
        "hcp_adamw_flat": (F_, F_ + 4096, F_ + 8192, F_ + 12288, 0, hyper.data_ptr(), 0.9, 0.999, 1e-8, 0.0, 1.0, None, 0.0, step.data_ptr(), S),
        "hcp_sumsq": (F_, 0, F_ + 64, S),
        "hcp_mse_loss": (F_, F_, 0, 1.0, F_ + 64, F_ + 128, S),
        "hcp_add_noise": (F_, F_, t.data_ptr(), F_, 0, 4, F_ + 64, S),
        "hcp_cast_f32_to_bf16": (F_, 0, B_, S),
        "hcp_geglu_fwd_bf16": (B_, 0, 8, B_ + 1024, S),
        "hcp_geglu_bwd_bf16": (B_, B_, 0, 8, B_ + 1024, S),
        "hcp_gelu_fwd_bf16": (B_, 0, 8, B_ + 1024, S),
        "hcp_gelu_bwd_bf16": (B_, B_, 0, 8, B_ + 1024, S),
        "hcp_quick_gelu_fwd_bf16": (B_, 0, 8, B_ + 1024, S),
        "hcp_quick_gelu_bwd_bf16": (B_, B_, 0, 8, B_ + 1024, S),
        "hcp_upsample2x_fwd_bf16": (B_, 0, 2, 2, 8, B_ + 1024, S),
        "hcp_upsample2x_bwd_bf16": (B_, 1, 0, 2, 8, B_ + 1024, S),
        "hcp_add_bf16": (B_, B_, 0, B_ + 1024, S),
        "hcp_sum_bf16_to_f32": (srcs, 2, 0, F_, S),
    }
    for name, args in cases.items():
        rc = rc_of(name, *args)
        assert rc == 0, f"{name}: rc={rc} ({_lib.lib().hcp_last_error_string().decode()})"
    assert _lib.launch_count == before
    assert int(step) == 0 and bool((f == 1.5).all())


def test_misaligned_buffers_refused_before_launch():
    """The bf16 vector kernels load and store 16 bytes at a time: a pointer off 16-byte alignment is refused, nothing launched."""
    b = torch.zeros(1 << 16, dtype=BF, device=DEV)
    f = torch.zeros(1 << 14, device=DEV)
    state = dropout_state(1, 0)
    B_, F_, S = b.data_ptr(), f.data_ptr(), stream_ptr()
    A, O = B_ + 2, B_ + 32768 + 2          # one bf16 element past alignment
    before = _lib.launch_count
    cases = [
        ("hcp_geglu_fwd_bf16", (A, 4, 8, B_ + 32768, S)), ("hcp_geglu_fwd_bf16", (B_, 4, 8, O, S)),
        ("hcp_geglu_bwd_bf16", (B_, A, 4, 8, B_ + 32768, S)), ("hcp_geglu_bwd_bf16", (B_, B_, 4, 8, O, S)),
        ("hcp_gelu_fwd_bf16", (A, 4, 8, B_ + 32768, S)), ("hcp_gelu_bwd_bf16", (B_, B_, 4, 8, O, S)),
        ("hcp_quick_gelu_fwd_bf16", (B_, 4, 8, O, S)), ("hcp_quick_gelu_bwd_bf16", (A, B_, 4, 8, B_ + 32768, S)),
        ("hcp_upsample2x_fwd_bf16", (A, 1, 2, 2, 8, B_ + 32768, S)), ("hcp_upsample2x_bwd_bf16", (B_, 1, 2, 2, 8, O, S)),
        ("hcp_add_bf16", (B_, A, 64, B_ + 32768, S)), ("hcp_add_bf16", (B_, B_, 64, O, S)),
        ("hcp_sum_bf16_to_f32", ((C.c_void_p * 2)(B_, A), 2, 64, F_, S)),
        ("hcp_sum_bf16_to_f32", ((C.c_void_p * 1)(B_), 1, 64, F_ + 4, S)),
        ("hcp_dropout_bf16", (A, 64, None, 0, None, 0, 1, 4, 64, 0.1, state.data_ptr(), 1, B_ + 32768, 64, S)),
        ("hcp_dropout_bf16", (B_, 64, A, 64, None, 0, 1, 4, 64, 0.1, state.data_ptr(), 1, B_ + 32768, 64, S)),
        ("hcp_dropout_bf16", (B_, 64, None, 0, F_ + 4, 64, 1, 4, 64, 0.1, state.data_ptr(), 1, B_ + 32768, 64, S)),
        ("hcp_dropout_bf16", (B_, 64, None, 0, None, 0, 1, 4, 64, 0.1, state.data_ptr(), 1, O, 64, S)),
    ]
    for name, args in cases:
        assert rc_of(name, *args) == HCP_ERR_INVALID, name
    assert _lib.launch_count == before
