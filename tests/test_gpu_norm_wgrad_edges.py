"""GPU tests of the normalisation, weight-gradient, repack and time-embedding / boundary kernels at their dispatch edges
(`pytest -m gpu`).

Every host-side planner these kernels go through is restated in tests/norm_wgrad_plan.py, and the cases below are chosen from it:
the three GroupNorm implementations (single-pass cluster kernel with 1 / 2 / 4 / 8 CTAs per image, two-pass 8-vector and pair
kernels, and the 16384-pixel shapes whose forward and backward take different ones), every LayerNorm instantiation, every tile
geometry of the tensor-core weight gradient.  Each kernel is called through its C ABI and compared with a float64 reference computed
from the bf16 operands it reads (tests/kernel_check.py), and every output lands in a canary buffer whose surroundings must stay
untouched.  Accumulating outputs (weight, bias and affine gradients) start at 0.5, so `got - 0.5` is what the kernel added.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:                # also run as a script: the forced two-pass GroupNorm leg below
    sys.path.insert(0, ROOT)

from kernel_check import CANARY, F32SIN, F32SUM, FWD, NORM, STAT, Canary, compare  # noqa: E402
from norm_wgrad_plan import (AFFINE_CASES, COLSUM_CASES, CONV_WGRAD_CASES, GN_BATCH_CASES, GN_CASES, GN_OFFSET_SHAPES,  # noqa: E402
                             GN_OFFSETS, GN_TWO_PASS_CASES, LN_CASES, REPACK_JOBS, SMALL_LINEAR_CASES, WGRAD_CASES, conv_box, gn_plan,
                             ln_plan, small_linear_dx_plan, wgrad_plan)

pytestmark = pytest.mark.gpu

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import GroupNormArgs, RepackJob, call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402,F401  (runtime and models import each other: models first)
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.ops import ConvPack, LinearPack  # noqa: E402
from hcp_diffusion_b200.runtime import _weight_2d, host_and_blocks  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
G = 32
EPS = 1e-5
SIN_ABS = 2e-4          # sinusoid: fp32 argument t * freq at t = 999, measured 6.5e-5 absolute


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def silu_grad(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


# ----------------------------------------------------------------------------------------------------------------------------------
# GroupNorm through hcp_groupnorm_{fwd,bwd}_bf16
# ----------------------------------------------------------------------------------------------------------------------------------
class GNProblem:
    """x = cat(x1, x2) [B, HW, C] bf16 with 32 groups; `offset` > 0 shifts group g by (-1)^g * offset standard deviations."""

    def __init__(self, B, HW, C1, C2, silu, seed=0, offset=0.0):
        C_ = C1 + C2
        gen = torch.Generator().manual_seed(seed)
        x = torch.randn(B, HW, C_, generator=gen)
        if offset:
            sign = 1.0 - 2.0 * (torch.arange(G) % 2)
            x = x + (offset * sign).repeat_interleave(C_ // G)
        else:
            x = 2 * x + 0.5
        x = x.to(BF).to(DEV)
        self.B, self.HW, self.C1, self.C2, self.C, self.silu = B, HW, C1, C2, C_, silu
        self.x1 = x[..., :C1].contiguous()
        self.x2 = x[..., C1:].contiguous() if C2 else None
        self.gamma = (1 + 0.2 * torch.randn(C_, generator=gen)).to(DEV)
        self.beta = (0.2 * torch.randn(C_, generator=gen)).to(DEV)
        self.dy = torch.randn(B, HW, C_, generator=gen).to(BF).to(DEV)
        self.add1 = torch.randn(B, HW, C1, generator=gen).to(BF).to(DEV)
        self.add2 = torch.randn(B, HW, C2, generator=gen).to(BF).to(DEV) if C2 else None

    def images(self, i0, i1):
        """The same problem restricted to images [i0, i1) (batch invariance)."""
        p = GNProblem.__new__(GNProblem)
        p.__dict__.update(self.__dict__)
        p.B = i1 - i0
        for k in ("x1", "x2", "dy", "add1", "add2"):
            t = getattr(self, k)
            setattr(p, k, None if t is None else t[i0:i1].contiguous())
        return p

    def args(self, stats):
        lib = _lib.lib()
        wsb = lib.hcp_groupnorm_workspace_bytes(self.B, self.HW, G)
        self.ws = torch.empty((max(wsb, 4) // 4,), dtype=F32, device=DEV)
        a = GroupNormArgs()
        a.x1, a.x2 = self.x1.data_ptr(), None if self.x2 is None else self.x2.data_ptr()
        a.B, a.HW, a.C1, a.C2, a.G = self.B, self.HW, self.C1, self.C2, G
        a.gamma, a.beta, a.eps, a.silu = self.gamma.data_ptr(), self.beta.data_ptr(), EPS, int(self.silu)
        a.stats, a.workspace, a.workspace_bytes = stats.data_ptr(), self.ws.data_ptr(), wsb
        return a

    def forward(self):
        """-> (y canary [B*HW, C], stats canary [1, B*G*2])"""
        y = Canary(self.B * self.HW, self.C, ld=self.C, col0=0)
        st = Canary(1, self.B * G * 2, dtype=F32)
        a = self.args(st.view)
        a.y = y.view.data_ptr()
        call("hcp_groupnorm_fwd_bf16", C.byref(a), stream_ptr())
        return y, st

    def backward(self, stats, with_add):
        """-> (dx1 canary, dx2 canary or None), reading the forward's statistics"""
        dx1 = Canary(self.B * self.HW, self.C1, ld=self.C1, col0=0)
        dx2 = Canary(self.B * self.HW, self.C2, ld=self.C2, col0=0) if self.C2 else None
        a = self.args(stats)
        a.dy = self.dy.data_ptr()
        if with_add:
            a.add1 = self.add1.data_ptr()
            a.add2 = None if self.add2 is None else self.add2.data_ptr()
        a.dx1, a.dx2 = dx1.view.data_ptr(), None if dx2 is None else dx2.view.data_ptr()
        call("hcp_groupnorm_bwd_bf16", C.byref(a), stream_ptr())
        return dx1, dx2

    def reference(self):
        """float64 y, mean, rstd [B, G] and dx = d(y . dy)/dx (without the residual-branch gradients)"""
        x = torch.cat([self.x1] + ([self.x2] if self.C2 else []), -1).to(F64).requires_grad_(True)
        B, HW, C_ = x.shape
        xg = x.view(B, HW, G, C_ // G)
        mean = xg.mean((1, 3), keepdim=True)
        var = (xg - mean).square().mean((1, 3), keepdim=True)
        rstd = (var + EPS).rsqrt()
        z = ((xg - mean) * rstd).view(B, HW, C_) * self.gamma.to(F64) + self.beta.to(F64)
        y = F.silu(z) if self.silu else z
        y.backward(self.dy.to(F64))
        return y.detach(), mean.detach().view(B, G), rstd.detach().view(B, G), x.grad


def check_stats(name, got, mean, rstd, mean_tol=STAT, rstd_tol=STAT):
    """got fp32 (mean, rstd) pairs; mean error in units of the standard deviation, rstd error relative"""
    got, mean, rstd = got.reshape(-1, 2).to(F64), mean.flatten(), rstd.flatten()
    em = float(((got[:, 0] - mean).abs() * rstd).max())
    er = float((got[:, 1] / rstd - 1).abs().max())
    print(f"{name}: mean err {em:.3e} sigma (<= {mean_tol:.1e}), rstd rel err {er:.3e} (<= {rstd_tol:.1e})")
    assert em <= mean_tol and er <= rstd_tol, f"{name}: statistics off (mean {em:.3e} sigma, rstd {er:.3e})"


def offset_stat_tols(k, centred):
    """Statistics bounds at means of k standard deviations.  An fp32 mean of k sigma is itself rounded to ~6e-8 k sigma (measured
    4.6e-6 sigma at k = 64).  GroupNorm takes the variance as E[x^2] - mean^2 in fp32, which cancels about 2 log2(k) bits: its rstd
    error grows as k^2 (measured on one H100: 5.5e-7 / 5.9e-6 / 5.4e-4 relative at k = 0 / 8 / 64); LayerNorm centres its second
    moment and keeps STAT (2.0e-7 at k = 64)."""
    return STAT * (1 + k / 8), STAT * (1 + k * k / 4) if not centred else STAT


def check_groupnorm(p: GNProblem, name: str, stat_tols=(STAT, STAT)):
    y, st = p.forward()
    yr, mean, rstd, dxr = p.reference()
    B, HW, C_ = p.B, p.HW, p.C
    compare(f"{name} y", y.view.reshape(B, HW, C_), yr, NORM, block=(128, 64))
    y.check(f"{name} y")
    check_stats(f"{name} stats", st.view, mean, rstd, *stat_tols)
    st.check(f"{name} stats")
    for with_add in (False, True):
        dx1, dx2 = p.backward(st.view, with_add)
        parts = [(dx1, dxr[..., :p.C1], p.add1, "dx1")] + ([(dx2, dxr[..., p.C1:], p.add2, "dx2")] if p.C2 else [])
        for can, ref, add, nm in parts:
            ref = ref + add.to(F64) if with_add else ref
            compare(f"{name} {nm}{' + add' if with_add else ''}", can.view.reshape(B, HW, -1), ref, NORM, block=(128, 64))
            can.check(f"{name} {nm}")
    return y, st


def gn_name(B, HW, C1, C2, silu, two_pass=False):
    f, b = gn_plan(HW, C1, C2, G, False, two_pass), gn_plan(HW, C1, C2, G, True, two_pass)
    geo = lambda q: q["path"] + (f"(S{q['S']} CB{q['CB']})" if q["path"] == "gnf" else f"(cg{q['cg']})")   # noqa: E731
    return f"gn B{B} HW{HW} {C1}+{C2} silu{int(silu)} fwd {geo(f)} bwd {geo(b)}"


@pytest.mark.parametrize("B,HW,C1,C2,silu", GN_CASES)
def test_groupnorm_paths(B, HW, C1, C2, silu):
    p = GNProblem(B, HW, C1, C2, silu, seed=B * 7 + HW)
    y, st = check_groupnorm(p, gn_name(B, HW, C1, C2, silu))
    # determinism: neither path uses atomics, so a repeated call gives the same bits
    y2, st2 = p.forward()
    assert torch.equal(y.view.view(torch.int16), y2.view.view(torch.int16)) and torch.equal(st.view, st2.view)
    d1, d2 = p.backward(st.view, True), p.backward(st.view, True)
    for a, b in zip(d1, d2):
        if a is not None:
            assert torch.equal(a.view.view(torch.int16), b.view.view(torch.int16)), "groupnorm backward changed on a repeated call"


@pytest.mark.parametrize("B,HW,C1,C2,silu", GN_BATCH_CASES)
def test_groupnorm_batch_invariance(B, HW, C1, C2, silu):
    """Image 1 of a batch of 3 and the same image alone: bit-identical y, statistics and dx on every path (the pixel chunking and
    cluster size depend on HW only)."""
    p = GNProblem(B, HW, C1, C2, silu, seed=5)
    one = p.images(1, 2)
    outs = []
    for q, sl in ((p, slice(HW, 2 * HW)), (one, slice(0, HW))):
        y, st = q.forward()
        dx1, dx2 = q.backward(st.view, True)
        k = (G * 2) if q is p else 0
        outs.append([y.view[sl].view(torch.int16), st.view[0, k:k + 2 * G], dx1.view[sl].view(torch.int16)] +
                    ([dx2.view[sl].view(torch.int16)] if dx2 is not None else []))
    assert all(torch.equal(a, b) for a, b in zip(*outs)), "image 1 differs between batch 3 and batch 1"


@pytest.mark.parametrize("offset", GN_OFFSETS)
@pytest.mark.parametrize("B,HW,C1,C2", GN_OFFSET_SHAPES)
def test_groupnorm_offset_stress(B, HW, C1, C2, offset):
    """Group means of 0, 8 and 64 standard deviations (alternating in sign) on each of the three paths.  y and dx keep the NORM
    bounds at every offset (the bf16 rounding of the output dominates); the statistics lose precision as k^2 (offset_stat_tols).
    The statistics bound is fitted to the measured growth at these three offsets; nothing is claimed beyond 64 sigma, where the
    fp32 E[x^2] - mean^2 keeps losing two bits per doubling of the offset and the outputs eventually leave NORM as well."""
    p = GNProblem(B, HW, C1, C2, True, seed=11, offset=offset)
    check_groupnorm(p, gn_name(B, HW, C1, C2, True) + f" offset {offset:g} sigma", offset_stat_tols(offset, centred=False))


def test_groupnorm_two_pass_kernels_at_single_pass_shapes():
    """HCP_GN_TWO_PASS (read once per process) forces the two-pass kernels: run the single-pass shapes through them in a child."""
    env = dict(os.environ, HCP_GN_TWO_PASS="1")
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "two-pass"]
    r = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    print(r.stdout[-20000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count("two-pass case ok") == len(GN_TWO_PASS_CASES)


# ----------------------------------------------------------------------------------------------------------------------------------
# LayerNorm through hcp_layernorm_{fwd,bwd}_bf16
# ----------------------------------------------------------------------------------------------------------------------------------
def check_layernorm(M, C_, offset=0.0, seed=0):
    plan = ln_plan(M, C_, sms())
    name = f"ln M{M} C{C_} NVPL{plan['nvpl']} {'pipelined' if plan['pipe'] else 'plain'} rpw{plan['rpw']}" + \
        (f" offset {offset:g} sigma" if offset else "")
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, C_, generator=gen)
    x = x + offset * (1.0 - 2.0 * (torch.arange(M) % 2))[:, None] if offset else 1.5 * x + 0.2
    x = x.to(BF).to(DEV)
    gamma = (1 + 0.2 * torch.randn(C_, generator=gen)).to(DEV)
    beta = (0.2 * torch.randn(C_, generator=gen)).to(DEV)
    dy = torch.randn(M, C_, generator=gen).to(BF).to(DEV)
    add = torch.randn(M, C_, generator=gen).to(BF).to(DEV)
    y = Canary(M, C_, ld=C_, col0=0)
    st = Canary(1, 2 * M, dtype=F32)
    call("hcp_layernorm_fwd_bf16", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), EPS, M, C_, st.view.data_ptr(), y.view.data_ptr(),
         stream_ptr())
    xr = x.to(F64).requires_grad_(True)
    mean = xr.mean(1, keepdim=True)
    rstd = ((xr - mean).square().mean(1, keepdim=True) + EPS).rsqrt()
    yr = (xr - mean) * rstd * gamma.to(F64) + beta.to(F64)
    yr.backward(dy.to(F64))
    compare(f"{name} y", y.view, yr.detach(), NORM, block=(plan["rpw"] * 8, C_))
    y.check(f"{name} y")
    check_stats(f"{name} stats", st.view, mean.detach().flatten(), rstd.detach().flatten(), *offset_stat_tols(offset, centred=True))
    st.check(f"{name} stats")
    for with_add in (False, True):
        dx = Canary(M, C_, ld=C_, col0=0)
        call("hcp_layernorm_bwd_bf16", x.data_ptr(), dy.data_ptr(), add.data_ptr() if with_add else None, gamma.data_ptr(),
             st.view.data_ptr(), M, C_, dx.view.data_ptr(), stream_ptr())
        ref = xr.grad + add.to(F64) if with_add else xr.grad
        compare(f"{name} dx{' + add' if with_add else ''}", dx.view, ref, NORM, block=(plan["rpw"] * 8, C_))
        dx.check(f"{name} dx")
    return plan


@pytest.mark.parametrize("M,C", LN_CASES)
def test_layernorm_instantiations(M, C):
    plan = check_layernorm(M, C)
    assert plan == ln_plan(M, C), f"this H100 has {sms()} SMs: the case no longer reaches the variant it was chosen for"


@pytest.mark.parametrize("offset", [8.0, 64.0])
@pytest.mark.parametrize("M,C", [(16389, 320), (300, 1280)])
def test_layernorm_offset_stress(M, C, offset):
    """Row means of 8 and 64 standard deviations: LayerNorm centres its second moment, so the offset costs nothing."""
    check_layernorm(M, C, offset=offset, seed=3)


# ----------------------------------------------------------------------------------------------------------------------------------
# GroupNorm / LayerNorm affine gradients and column sums (hcp_norm_affine_grad_bf16, hcp_colsum_bf16)
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,HW,C1,C2,groups,silu", AFFINE_CASES)
def test_norm_affine_grad(B, HW, C1, C2, groups, silu):
    C_ = C1 + C2
    rows = B * HW
    x = rnd(rows, C_, scale=1.5, seed=1) + 0.3
    x1, x2 = x[:, :C1].contiguous(), x[:, C1:].contiguous() if C2 else None
    dy = rnd(rows, C_, seed=2)
    gamma, beta = 1 + rnd(C_, scale=0.2, seed=3, dtype=F32), rnd(C_, scale=0.2, seed=4, dtype=F32)
    xd = x.to(F64)
    if groups:
        xg = xd.view(B, HW, groups, C_ // groups)
        mean = xg.mean((1, 3))
        rstd = (xg.var((1, 3), unbiased=False) + EPS).rsqrt()
        stats = torch.stack([mean, rstd], -1).to(F32).contiguous()                 # [B, groups, 2]
        m_r = stats[..., 0].to(F64).repeat_interleave(C_ // groups, 1).repeat_interleave(HW, 0)
        r_r = stats[..., 1].to(F64).repeat_interleave(C_ // groups, 1).repeat_interleave(HW, 0)
    else:
        mean = xd.mean(1)
        rstd = (xd.var(1, unbiased=False) + EPS).rsqrt()
        stats = torch.stack([mean, rstd], -1).to(F32).contiguous()                 # [rows, 2]
        m_r, r_r = stats[:, :1].to(F64), stats[:, 1:].to(F64)
    h = (xd - m_r) * r_r
    dz = dy.to(F64)
    if silu:
        dz = dz * silu_grad(gamma.to(F64) * h + beta.to(F64))
    ref_g, ref_b = (dz * h).sum(0), dz.sum(0)
    dg, db = Canary(1, C_, dtype=F32), Canary(1, C_, dtype=F32)
    dg.view.fill_(0.5)
    db.view.fill_(0.5)
    call("hcp_norm_affine_grad_bf16", x1.data_ptr(), None if x2 is None else x2.data_ptr(), C1, C2, dy.data_ptr(), stats.data_ptr(),
         gamma.data_ptr(), beta.data_ptr(), rows, HW if groups else 0, groups, int(silu), dg.view.data_ptr(), db.view.data_ptr(),
         stream_ptr())
    name = f"affine B{B} HW{HW} {C1}+{C2} groups{groups} silu{int(silu)}"
    compare(f"{name} dgamma", dg.view - 0.5, ref_g.view(1, -1), F32SUM, block=(1, 64))
    compare(f"{name} dbeta", db.view - 0.5, ref_b.view(1, -1), F32SUM, block=(1, 64))
    dg.check(f"{name} dgamma")
    db.check(f"{name} dbeta")


@pytest.mark.parametrize("M,N,ld,rpg,scale", COLSUM_CASES)
def test_colsum(M, N, ld, rpg, scale):
    buf = rnd(M, ld + 8, seed=1)
    x = buf[:, 8:8 + N]                                     # a column slice at a 16-byte offset, row pitch ld + 8
    groups = M // (rpg or M)
    out = Canary(groups, N, dtype=F32)                       # ldo = N + 64
    out.view.fill_(0.5)
    call("hcp_colsum_bf16", x.data_ptr(), ld + 8, M, N, rpg, scale, out.view.data_ptr(), out.ld, stream_ptr())
    ref = x.to(F64).view(groups, M // groups, N).sum(1) * scale
    compare(f"colsum M{M} N{N} ld{ld + 8} rows/group {rpg or M} scale {scale}", out.view - 0.5, ref, F32SUM, block=(1, 64))
    out.check("colsum")


# ----------------------------------------------------------------------------------------------------------------------------------
# tensor-core weight gradients (hcp_wgrad_bf16, hcp_wgrad_conv3x3_bf16)
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,j_cols,n_cols", WGRAD_CASES)
def test_linear_wgrad(M, j_cols, n_cols):
    """dW[j, n] += scale * sum_m dY[m, j] X[m, n]: column slices of dY and X (row pitches wider than the data) into a column slice
    of a wider dW (ld_j != n_cols)."""
    plan = wgrad_plan(M, j_cols, n_cols, sms())
    sbuf, xbuf = rnd(M, j_cols + 24, seed=1), rnd(M, n_cols + 16, seed=2)
    S, X = sbuf[:, 8:8 + j_cols], xbuf[:, 8:8 + n_cols]
    scale = 0.25 if M % 2 else 1.0
    dst = Canary(j_cols, n_cols, ld=(n_cols + 7) // 8 * 8 + 64, dtype=F32)
    dst.view.fill_(0.5)
    call("hcp_wgrad_bf16", S.data_ptr(), sbuf.shape[1], j_cols, X.data_ptr(), xbuf.shape[1], n_cols, M, scale, dst.view.data_ptr(),
         dst.ld, 1, stream_ptr())
    ref = scale * S.to(F64).t() @ X.to(F64)
    compare(f"wgrad M{M} j{j_cols} n{n_cols} SN{plan['sn']} splits{plan['splits']}x{plan['tiles_per_cta']}", dst.view - 0.5, ref, F32SUM,
            block=(plan["sn"], 128))
    dst.check("wgrad dW")


def conv_wgrad_ref(x, dy, stride):
    """float64 dW [Cout, Cin, 3, 3] of a 3x3 / pad 1 convolution: one GEMM per tap over the shifted input. x [B, H, W, Cin],
    dy [B, Ho, Wo, Cout]."""
    B, Ho, Wo, Cout = dy.shape
    Cin = x.shape[-1]
    xp = F.pad(x.to(F64), (0, 0, 1, 1, 1, 1))
    d = dy.to(F64).reshape(-1, Cout)
    dw = torch.empty(Cout, Cin, 3, 3, dtype=F64, device=x.device)
    for kh in range(3):
        for kw in range(3):
            xs = xp[:, kh:kh + stride * Ho:stride, kw:kw + stride * Wo:stride]
            dw[:, :, kh, kw] = d.t() @ xs.reshape(-1, Cin)
    return dw


@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", CONV_WGRAD_CASES)
def test_conv3x3_wgrad(B, H, W, Cin, Cout, stride):
    geo = conv_box(B, H, W, stride)
    Ho, Wo = H // stride, W // stride
    x = rnd(B, H, W, Cin, seed=1)
    dy = rnd(B, Ho, Wo, Cout, seed=2)
    dw = Canary(1, Cout * Cin * 9, dtype=F32)
    dw.view.fill_(0.5)
    call("hcp_wgrad_conv3x3_bf16", dy.data_ptr(), Cout, x.data_ptr(), B, H, W, Cin, stride, 1.0, dw.view.data_ptr(), stream_ptr())
    ref = conv_wgrad_ref(x, dy, stride)
    sn = 128 if Cout > 64 else 64
    got = (dw.view - 0.5).view(Cout, Cin, 3, 3).permute(2, 3, 0, 1).reshape(9, Cout, Cin)
    compare(f"conv wgrad B{B} {H}x{W} {Cin}->{Cout} s{stride} box {geo['bw']}x{geo['bh']}x{geo['bnimg']}", got,
            ref.permute(2, 3, 0, 1).reshape(9, Cout, Cin), F32SUM, block=(sn, 128))
    dw.check("conv wgrad dW")


# ----------------------------------------------------------------------------------------------------------------------------------
# per-step repack of the trained weights (hcp_repack_weights): bit for bit
# ----------------------------------------------------------------------------------------------------------------------------------
def test_repack_weights_bit_exact():
    """All jobs of REPACK_JOBS in one launch.  Every destination starts as all-ones canary bits; afterwards it must equal that
    canary with exactly the job's rows / columns replaced by the round-to-nearest-even bf16 of the fp32 masters (torch's
    `.to(bfloat16)`, as LinearPack builds W / WT), the ConvPack operands of the same masters, or the fp32 bias."""
    def canary(*shape, dtype=BF):
        return torch.full(shape, CANARY, dtype=torch.int16 if dtype == BF else torch.int32, device=DEV).view(dtype)

    jobs, keep, outs = [], [], {}           # outs: name -> (destination, expected bits)
    for i, (kind, rows, K, o0, n_tot, flip) in enumerate(REPACK_JOBS):
        j = RepackJob()
        j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = kind, rows, K, o0, n_tot, flip
        if kind in (0, 3):
            src = rnd(rows, K, seed=20 + i, dtype=F32)
            name = f"kind {kind} K{K} n_tot{n_tot}"           # the hosts of one fused group share their destinations
            if name + " W" not in outs:
                n = n_tot if kind == 0 else o0 + rows + 11
                outs[name + " W"] = (canary(n, K), canary(n, K))
                if kind == 0:
                    outs[name + " WT"] = (canary(K, n), canary(K, n))
            d0, e0 = outs[name + " W"]
            e0[o0:o0 + rows] = src.to(BF)
            j.dst0, j.dst1 = d0.data_ptr(), None
            if kind == 0:
                d1, e1 = outs[name + " WT"]
                e1[:, o0:o0 + rows] = src.to(BF).t()
                j.dst1 = d1.data_ptr()
        elif kind == 1:
            src = rnd(rows, K, 3, 3, seed=20 + i, dtype=F32)
            pack = ConvPack(src, None, 1 if flip else 2)
            for nm, op in (("W", pack.W), ("Wd", pack.Wd)):
                d, e = canary(op.numel() + 24), canary(op.numel() + 24)
                e[8:8 + op.numel()] = op.flatten()
                outs[f"conv {rows}x{K} flip{flip} {nm}"] = (d, e)
            j.dst0 = outs[f"conv {rows}x{K} flip{flip} W"][0][8:].data_ptr()
            j.dst1 = outs[f"conv {rows}x{K} flip{flip} Wd"][0][8:].data_ptr()
        else:
            src = rnd(rows, seed=20 + i, dtype=F32)
            d, e = canary(o0 + rows + 13, dtype=F32), canary(o0 + rows + 13, dtype=F32)
            e[o0:o0 + rows] = src
            outs[f"bias {rows} at {o0}"] = (d, e)
            j.dst0, j.dst1 = d.data_ptr(), None
        j.src = src.data_ptr()
        keep.append(src)
        jobs.append(j)
    arr = (RepackJob * len(jobs))(*jobs)
    table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(DEV)
    call("hcp_repack_weights", table.data_ptr(), len(jobs), stream_ptr())
    bad = {}
    for name, (d, e) in outs.items():
        bits = torch.int16 if d.dtype == BF else torch.int32
        bad[name] = int((d.view(bits) != e.view(bits)).sum())
        print(f"repack {name}: {bad[name]} of {d.numel()} elements differ")
    assert not any(bad.values()), f"repack destinations differ from the operands of the fp32 masters: {bad}"


def full_ft_unet(spec):
    """A UNet of `spec` with every layer trained (DreamBooth.yaml / FT_sdxl.yaml: `unet: [{layers: ['']}]`)."""
    down = tuple("CrossAttnDownBlock2D" if a else "DownBlock2D" for a in spec.down_has_attn)
    up = tuple("CrossAttnUpBlock2D" if a else "UpBlock2D" for a in spec.up_has_attn)
    unet = UNet2DConditionModel(
        sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
        cross_attention_dim=spec.cross_attention_dim, down_block_types=down, up_block_types=up,
        transformer_layers_per_block=spec.transformer_depth, use_linear_projection=spec.use_linear_projection,
        addition_embed_type="text_time" if spec.addition_time_embed_dim else None, addition_time_embed_dim=spec.addition_time_embed_dim,
        projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)
    unet.load_state_dict(U.init_params(spec))
    unet = unet.to(DEV).requires_grad_(False).eval()
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-3, "layers": [""]}], None)
    assert lora.empty() and all(p.requires_grad for p in unet.parameters())
    return unet, groups


def trained_operands(unet):
    """[(name, operand the kernels read, the same operand built afresh from the current fp32 masters, master weights it covers)]:
    every fused linear group (LinearPack W / WT / bias of the concatenated hosts), every 3x3 convolution (ConvPack W / Wd / bias), the
    time-embedding MLP, the stacked time_emb_proj rows and biases, the additional embedding (SDXL) and the boundary convolutions."""
    out = []
    for i, g in enumerate(unet.linear_groups()):
        hosts = [host_and_blocks(ch)[0] for ch in g.children]
        w = torch.cat([_weight_2d(h) for h in hosts], 0)
        bias = None                                      # as LinearGroup.prepare: no fused bias when no host has one
        if any(h.bias is not None for h in hosts):
            bias = torch.cat([h.bias if h.bias is not None else torch.zeros(h.weight.shape[0], device=DEV) for h in hosts])
        fresh = LinearPack(w, bias, g.pack.k_splits)
        ws = [h.weight for h in hosts]
        out += [(f"linear group {i} W", g.pack.W, fresh.W, ws), (f"linear group {i} WT", g.pack.WT, fresh.WT, []),
                (f"linear group {i} bias", g.pack.bias, fresh.bias, [])]
    for i, g in enumerate(unet.conv_groups()):
        conv = host_and_blocks(g.conv)[0]
        fresh = ConvPack(conv.weight, conv.bias, conv.stride[0])
        out += [(f"conv {i} s{conv.stride[0]} W", g.pack.W, fresh.W, [conv.weight]), (f"conv {i} Wd", g.pack.Wd, fresh.Wd, []),
                (f"conv {i} bias", g.pack.bias, fresh.bias, [])]
    rt = unet.__dict__["_rt"]
    te, resnets = unet.time_embedding, unet.resnets_in_order()
    projs = [unet._temb_host(r) for r in resnets]
    out += [("time linear_1 W", rt.w1, te.linear_1.weight.to(BF), [te.linear_1.weight]), ("time linear_1 b", rt.b1, te.linear_1.bias, []),
            ("time linear_2 W", rt.w2, te.linear_2.weight.to(BF), [te.linear_2.weight]), ("time linear_2 b", rt.b2, te.linear_2.bias, []),
            ("time_emb_proj rows", rt.wp, torch.cat([p.weight for p in projs]).to(BF), [p.weight for p in projs]),
            ("time_emb_proj biases", rt.bp, torch.cat([p.bias for p in projs]), [])]
    if hasattr(unet, "add_embedding"):
        ae = unet.add_embedding
        out += [("add linear_1 W", rt.add.w1, ae.linear_1.weight.to(BF), [ae.linear_1.weight]), ("add linear_1 b", rt.add.b1, ae.linear_1.bias, []),
                ("add linear_2 W", rt.add.w2, ae.linear_2.weight.to(BF), [ae.linear_2.weight]), ("add linear_2 b", rt.add.b2, ae.linear_2.bias, [])]
    out += [("conv_in W", rt.w_in, unet.conv_in.weight.permute(1, 2, 3, 0), [unet.conv_in.weight]), ("conv_in b", rt.b_in, unet.conv_in.bias, []),
            ("conv_out W", rt.w_out, unet.conv_out.weight.permute(2, 3, 0, 1), [unet.conv_out.weight]), ("conv_out b", rt.b_out, unet.conv_out.bias, [])]
    assert all((op is None) == (fresh is None) for _, op, fresh, _ in out), [name for name, op, fresh, _ in out if (op is None) != (fresh is None)]
    return [e for e in out if e[1] is not None]


@pytest.mark.parametrize("spec_name,optimizer", [("TINY", "adamw"), ("TINY_XL", "adafactor")])
def test_full_finetune_operands_equal_fresh_packs_after_a_step(spec_name, optimizer):
    """One optimizer step of a full fine-tune, then the next forward: every operand the kernels read -- each LinearPack's W / WT /
    fused bias, each ConvPack's W / Wd (flipped for stride 1, not for stride 2) / bias, the time-embedding and additional-embedding
    operands, the stacked time_emb_proj rows and biases -- must equal, bit for bit, the same operand built afresh from the updated
    fp32 masters.  This checks the host-side job tables (row offsets of fused q|k|v and k|v hosts, n_tot, flip, the bias jobs, the
    time-embedding jobs) that drive hcp_repack_weights, not only the kernel."""
    spec = getattr(U, spec_name)
    unet, groups = full_ft_unet(spec)
    step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=False, optimizer=optimizer)
    lat, noise, t, ehs = (v.to(DEV) for v in U.synthetic_batch(2, spec))
    added = U.synthetic_added_cond(2, spec)
    added = None if added is None else {k: v.to(DEV) for k, v in added.items()}
    step.step(lat, noise, t, ehs, added)                   # forward (operands of the initial masters), backward, optimizer
    before = [(name, op.clone()) for name, op, _, _ in trained_operands(unet)]
    step._forward_backward(lat, noise, t, ehs, added)      # the next forward repacks from the updated masters
    torch.cuda.synchronize()
    ops_now = trained_operands(unet)
    covered = {id(w) for *_, ws in ops_now for w in ws}
    weights = [m.weight for m in unet.modules() if isinstance(m, (torch.nn.Linear, torch.nn.Conv2d))]
    assert all(id(w) in covered for w in weights), "a trained linear / convolution weight has no operand check"
    bad, moved = [], 0
    for (name, op, fresh, _), (_, old) in zip(ops_now, before):
        fresh = fresh.detach().contiguous().to(op.dtype)
        bits = torch.int16 if op.dtype == BF else torch.int32
        assert op.shape == fresh.shape, f"{name}: {tuple(op.shape)} != {tuple(fresh.shape)}"
        n = int((op.view(bits) != fresh.view(bits)).sum())
        moved += int(not torch.equal(old.view(bits), op.view(bits)))
        if n:
            bad.append((name, n, op.numel()))
    print(f"{spec_name}: {len(ops_now)} operands, {moved} changed by the step, mismatches {bad}")
    assert not bad, f"operands differ from fresh packs of the updated masters: {bad}"
    assert moved >= 0.9 * len(ops_now), "the step left most operands unchanged: the check would not see a stale repack"


# ----------------------------------------------------------------------------------------------------------------------------------
# time-embedding and boundary kernels
# ----------------------------------------------------------------------------------------------------------------------------------
def flat_f32(n, fill=float("nan")):
    """n fp32 outputs with 16 canary elements on each side: (buffer, view)"""
    buf = torch.full((n + 32,), -1, dtype=torch.int32, device=DEV).view(F32)
    v = buf[16:16 + n]
    if fill == fill:
        v.fill_(fill)
    return buf, v


def flat_check(name, buf, n):
    bits = buf.view(torch.int32)
    stray = int((bits[:16] != -1).sum() + (bits[16 + n:] != -1).sum())
    assert stray == 0, f"{name}: {stray} elements outside the output were written"


def sinusoid64(t, dim):
    half = dim // 2
    a = t.to(F64)[:, None] * torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64, device=t.device) / half)
    return torch.cat([a.cos(), a.sin()], -1)


@pytest.mark.parametrize("M,K,N,in_mode,out_silu", [(1, 320, 1283, 2, 1), (16, 320, 13, 2, 0), (16, 1280, 1283, 1, 0),
                                                    (5, 2816, 1280, 0, 1), (3, 256, 1281, 1, 1)])
def test_skinny_linear(M, K, N, in_mode, out_silu):
    """y = f(x) W^T + b for M <= 16 rows, one warp per output column, eight per block (N % 8 != 0: a part-filled last block)."""
    x = (torch.tensor([0.0, 1.0, 999.0, 500.0, 17.0] * 4)[:M].to(DEV) if in_mode == 2 else rnd(M, K, seed=1, dtype=F32))
    w = rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    b = rnd(N, scale=0.3, seed=3, dtype=F32)
    buf, y = flat_f32(M * N)
    call("hcp_skinny_linear", x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, in_mode, out_silu, y.data_ptr(), stream_ptr())
    xi = sinusoid64(x, K) if in_mode == 2 else x.to(F64)
    if in_mode == 1:
        xi = F.silu(xi)
    ref = xi @ w.to(F64).t() + b.to(F64)
    if out_silu:
        ref = F.silu(ref)
    compare(f"skinny M{M} K{K} N{N} in_mode{in_mode} silu{out_silu}", y.view(M, N), ref,
            F32SUM if in_mode != 2 else F32SIN, block=(M, 8))
    flat_check("skinny y", buf, M * N)


@pytest.mark.parametrize("M,N,K", [c[:3] for c in SMALL_LINEAR_CASES])
def test_small_linear_bwd(M, N, K):
    """dx = dy W over 16-row blocks, dW += dy^T x, db += colsum(dy); dy a column slice (ldy = N + 64).  (64, 40960, 1280) is the case
    whose dx grid doubles n_chunk (small_linear_dx_plan); it runs dx alone."""
    plan = small_linear_dx_plan(M, N, K)
    with_dw = {c[:3]: c[3] for c in SMALL_LINEAR_CASES}[(M, N, K)]
    dyb = rnd(M, N + 64, seed=1, dtype=F32)
    dy = dyb[:, 32:32 + N]
    x = rnd(M, K, seed=2, dtype=F32)
    w = rnd(N, K, scale=1 / math.sqrt(N), seed=3)
    dxb, dx = flat_f32(M * K)
    dwb, dw = flat_f32(N * K, 0.5) if with_dw else (None, None)
    dbb, db = flat_f32(N, 0.5) if with_dw else (None, None)
    call("hcp_small_linear_bwd_f32", dy.data_ptr(), N + 64, x.data_ptr(), w.data_ptr(), M, N, K, dx.data_ptr(),
         dw.data_ptr() if with_dw else None, db.data_ptr() if with_dw else None, stream_ptr())
    d = dy.to(F64)
    dx_ref = torch.zeros(M, K, dtype=F64, device=DEV)
    for n0 in range(0, N, 8192):                          # float64 copies of W one slice at a time
        dx_ref += d[:, n0:n0 + 8192] @ w[n0:n0 + 8192].to(F64)
    name = f"small linear bwd M{M} N{N} K{K} n_chunk {plan['n_chunk']}"
    compare(f"{name} dx", dx.view(M, K), dx_ref, F32SUM, block=(16, 128))
    flat_check(f"{name} dx", dxb, M * K)
    if with_dw:
        compare(f"{name} dW", (dw - 0.5).view(N, K), d.t() @ x.to(F64), F32SUM, block=(128, 128))
        compare(f"{name} db", (db - 0.5).view(1, N), d.sum(0, keepdim=True), F32SUM, block=(1, 128))
        flat_check(f"{name} dW", dwb, N * K)
        flat_check(f"{name} db", dbb, N)


def test_sinusoid_matches_oracle_timestep_embedding():
    """hcp_sinusoid_f32 at t in {0, 1, 999} (and SDXL's six time ids per row, written at a row pitch wider than 6 x 256) against
    oracle.unet_ref.timestep_embedding and its float64 restatement."""
    t = torch.tensor([0.0, 1.0, 999.0, 1024.0, 512.0, 1.0], device=DEV)
    for dim, per_row, ld in ((320, 1, 320), (256, 6, 6 * 256 + 64)):
        rows = (t.numel() + per_row - 1) // per_row
        buf, out = flat_f32(rows * ld)
        call("hcp_sinusoid_f32", t.data_ptr(), t.numel(), dim, per_row, out.data_ptr(), ld, stream_ptr())
        got = out.view(rows, ld)[:, :per_row * dim].reshape(-1, dim)
        ref = sinusoid64(t, dim)
        orc = U.timestep_embedding(t.cpu(), dim).to(DEV)
        e64, eor = float((got.to(F64) - ref).abs().max()), float((got - orc).abs().max())
        print(f"sinusoid dim{dim} per_row{per_row}: max abs vs float64 {e64:.3e}, vs oracle {eor:.3e} (<= {SIN_ABS:.0e})")
        assert e64 <= SIN_ABS and eor <= SIN_ABS
        if ld > per_row * dim:
            assert torch.isnan(out.view(rows, ld)[:, per_row * dim:]).all(), "sinusoid wrote past its row"
        flat_check("sinusoid", buf, rows * ld)


@pytest.mark.parametrize("B,H,W,Cin,Cwide", [(3, 12, 12, 4, 320), (1, 128, 128, 4, 320), (2, 8, 8, 3, 64)])
def test_boundary_convolutions(B, H, W, Cin, Cwide):
    """conv_in (fp32 NCHW latent -> bf16 NHWC), conv_out (bf16 NHWC -> fp32 NCHW, 4 channels) and its input gradient, and both
    boundary weight gradients.  B*H*W = 432 is not a multiple of the 128-pixel chunk of the weight gradients: chunks span two
    images.  Cin = 3 (conv_in, its weight gradient and conv_out's weight gradient accept fewer than 4 narrow channels)."""
    lat = rnd(B, Cin, H, W, seed=1, dtype=F32)
    w_in = rnd(Cwide, Cin, 3, 3, scale=0.2, seed=2, dtype=F32)
    b_in = rnd(Cwide, scale=0.3, seed=3, dtype=F32)
    y = Canary(B * H * W, Cwide, ld=Cwide, col0=0)
    call("hcp_conv_in_f32", lat.data_ptr(), w_in.permute(1, 2, 3, 0).contiguous().data_ptr(), b_in.data_ptr(), B, Cin, H, W, Cwide,
         y.view.data_ptr(), stream_ptr())
    ref = F.conv2d(lat.to(F64), w_in.to(F64), b_in.to(F64), padding=1).permute(0, 2, 3, 1).reshape(-1, Cwide)
    name = f"B{B} {H}x{W} narrow{Cin} wide{Cwide}"
    compare(f"conv_in {name}", y.view, ref, FWD, block=(128, 64))
    y.check("conv_in y")
    # conv_in weight gradient: dh bf16 NHWC
    dh = rnd(B, H, W, Cwide, seed=4)
    dwb, dw = flat_f32(Cwide * Cin * 9, 0.5)
    dbb, db = flat_f32(Cwide, 0.5)
    call("hcp_conv_in_wgrad_f32", dh.data_ptr(), lat.data_ptr(), B, Cin, H, W, Cwide, dw.data_ptr(), db.data_ptr(), stream_ptr())
    dwr = conv_wgrad_ref(lat.permute(0, 2, 3, 1), dh, 1)
    compare(f"conv_in wgrad {name}", (dw - 0.5).view(Cwide, Cin * 9), dwr.reshape(Cwide, Cin * 9), F32SUM, block=(64, 9))
    compare(f"conv_in bias grad {name}", (db - 0.5).view(1, -1), dh.to(F64).sum((0, 1, 2)).view(1, -1), F32SUM, block=(1, 64))
    flat_check("conv_in wgrad", dwb, Cwide * Cin * 9)
    flat_check("conv_in bias grad", dbb, Cwide)
    # conv_out (4 output channels) forward and input gradient; its weight gradient with Cin narrow channels
    act = rnd(B, H, W, Cwide, seed=5)
    w_out = rnd(4, Cwide, 3, 3, scale=1 / math.sqrt(9 * Cwide), seed=6, dtype=F32)
    b_out = rnd(4, scale=0.3, seed=7, dtype=F32)
    ob, out = flat_f32(B * 4 * H * W)
    wtap = w_out.permute(2, 3, 0, 1).contiguous()
    call("hcp_conv_out_f32", act.data_ptr(), wtap.data_ptr(), b_out.data_ptr(), B, H, W, Cwide, 4, out.data_ptr(), stream_ptr())
    ar = act.to(F64).permute(0, 3, 1, 2)
    ref = F.conv2d(ar, w_out.to(F64), b_out.to(F64), padding=1)
    compare(f"conv_out {name}", out.view(B * 4, H * W), ref.reshape(B * 4, H * W), F32SUM, block=(4, 128))
    flat_check("conv_out y", ob, B * 4 * H * W)
    dy = rnd(B, 4, H, W, seed=8, dtype=F32)
    dx = Canary(B * H * W, Cwide, ld=Cwide, col0=0)
    call("hcp_conv_out_dgrad_f32", dy.data_ptr(), wtap.data_ptr(), B, H, W, Cwide, 4, dx.view.data_ptr(), stream_ptr())
    dxr = torch.nn.grad.conv2d_input(ar.shape, w_out.to(F64), dy.to(F64), padding=1).permute(0, 2, 3, 1).reshape(-1, Cwide)
    compare(f"conv_out dgrad {name}", dx.view, dxr, FWD, block=(128, 64))
    dx.check("conv_out dgrad")
    dyn = rnd(B, Cin, H, W, seed=9, dtype=F32)
    dwb2, dw2 = flat_f32(Cin * Cwide * 9, 0.5)
    dbb2, db2 = flat_f32(Cin, 0.5)
    call("hcp_conv_out_wgrad_f32", dyn.data_ptr(), act.data_ptr(), B, H, W, Cwide, Cin, dw2.data_ptr(), db2.data_ptr(), stream_ptr())
    dwr2 = conv_wgrad_ref(act, dyn.permute(0, 2, 3, 1), 1)
    compare(f"conv_out wgrad {name}", (dw2 - 0.5).view(Cin, Cwide * 9), dwr2.reshape(Cin, Cwide * 9), F32SUM, block=(Cin, 9 * 64))
    compare(f"conv_out bias grad {name}", (db2 - 0.5).view(1, -1), dyn.to(F64).sum((0, 2, 3)).view(1, -1), F32SUM, block=(1, Cin))
    flat_check("conv_out wgrad", dwb2, Cin * Cwide * 9)
    flat_check("conv_out bias grad", dbb2, Cin)


if __name__ == "__main__":
    # child of test_groupnorm_two_pass_kernels_at_single_pass_shapes: HCP_GN_TWO_PASS is set for this whole process
    assert sys.argv[1:] == ["two-pass"] and os.environ.get("HCP_GN_TWO_PASS")
    torch.cuda.set_device(0)
    for case in GN_TWO_PASS_CASES:
        check_groupnorm(GNProblem(*case, seed=case[0] * 7 + case[1]), gn_name(*case, two_pass=True))
        print("two-pass case ok", flush=True)
