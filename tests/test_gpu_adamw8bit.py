"""AdamW8bit on the GPU (`pytest -m gpu`): hcp_adamw8bit_flat against the fp32 restatement in tests/adamw8bit_ref.py at its edges,
the training step with optimizer='adamw8bit' against oracle.step_ref.ReferenceLoop running adamw8bit_ref.AdamW8bit, and the
entrypoint on a tiny copy of cfgs/train/ft_adamw8bit_sdxl_synthetic.yaml.

Kernel: four steps from the kernel's own state (random codes and scales to start), each restated from the exact fp32 / uint8
values the kernel read, with the clip factor computed as the kernel computes it.  The kernel and the restatement round every
operation of the moment update on its own, so the checks are:

                                                                  measured worst                 bound
  new absmax                                                      exact                          exact
  new codes                                                       0 mismatches                   only within A8_TIE_ULPS of a midpoint
  32-bit m', v' / (|m_ref| + 1e-30)                               0 (bit-exact)                  A8_M32
  p': (|p' - p_ref| - ulp(p_ref)) / |p_ref - p|                   2.22e-7                        A8_P = 6e-7
      (the bias corrections' powf is not correctly rounded on
      either side; up to 16 ulp of p' where |p'| is far below
      the update)
  an 8-bit p' whose gradient is not finite                        exact                          exact

Codes within 2 ulp of a midpoint over both tables and four steps: 6 and 41, none of them different.

Training step: the update (after - before) of each model is compared with the reference's by its direction cosine.  Adam's early
steps are close to sign steps, and bf16 noise in the gradient moves the 8-bit codes across a midpoint here and there, so the bound
sits under the worst cosine measured.  Numbers measured on one H100 80GB HBM3 at a 700 W power limit.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200 import adamw8bit as A  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

import adamw8bit_ref as R  # noqa: E402
import clip_ref as CR  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HCP_ERR_INVALID = -1
F32 = np.float32

A8_M32 = 2.4e-7                 # 32-bit m', v': 2 fp32 ulp (the arithmetic is the restatement's, so 0 is expected)
A8_P = 6e-7                     # p': (|p' - p_ref| - 1 ulp) / |p_ref - p|; measured 2.07e-7 / 2.22e-7 (blocks8 / mixed)
A8_TIE_ULPS = 2.0               # a code may differ from the restatement's only this close (fp32 ulps of x) to a midpoint
COS = 0.99                      # update cosine per model; measured 0.9976 / 0.9956 (LoRA, clip on / off), 0.9956 (full
                                # fine-tune), 0.9969 / 0.9969 (UNet / text-encoder adapters of the joint step)


def measured(name: str, value: float, bound: float, above: bool = False) -> None:
    print(f"MEASURED {name}: {value:.6e} ({'>=' if above else '<='} {bound:.2e})")
    assert (value >= bound) if above else (value <= bound), f"{name}: {value:.6e} vs {bound:.2e}"


def kernel_scale(gscale: float, sumsq: float, max_norm: float) -> np.float32:
    """grad_scale x clip as the kernel computes it (a8_grad_scale: every operation rounded to fp32 on its own)."""
    gs, mn = F32(gscale), F32(max_norm)
    clip = F32(1.0)
    if mn > 0:
        norm = F32(F32(np.sqrt(F32(sumsq))) * gs)
        clip = np.fmin(F32(1.0), F32(mn / F32(norm + F32(1e-6))))
    return F32(gs * clip)


class Table:
    """Tensors of `numels` packed in a flat buffer as FlatParams packs them (16-byte aligned, from element 4, so no tensor starts at
    a multiple of 256), tensor i in group i % ngroups, the state of adamw8bit.Layout; every buffer has canary room after it."""

    def __init__(self, numels, min8, ngroups=3, seed=0):
        self.offsets, off = [], 4
        for n in numels:
            self.offsets.append(off)
            off += (n + 3) // 4 * 4
        self.numels, self.n, self.ngroups = list(numels), off, ngroups
        self.lay = lay = A.Layout(numels, self.offsets, [i % ngroups for i in range(len(numels))], min8)
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.p = torch.randn(self.n + 16, generator=gen, device=DEV)
        self.g = torch.zeros(self.n + 16, device=DEV)
        # start from an arbitrary valid state: random codes and positive scales, random fp32 m and v >= 0
        self.codes = torch.randint(0, 256, (2 * lay.code_bytes + 64,), generator=gen, device=DEV, dtype=torch.uint8)
        self.absmax = torch.rand(2 * lay.nblocks + 16, generator=gen, device=DEV) * 1e-2
        self.state32 = torch.randn(2 * lay.small_numel + 16, generator=gen, device=DEV) * 1e-3
        self.state32[lay.small_numel:2 * lay.small_numel].abs_().mul_(1e-3)
        self.maps = A.maps().to(DEV)
        to_dev = lambda a: torch.from_numpy(a.view(np.uint8).copy()).to(DEV)      # noqa: E731
        self.tensors_dev, self.items_dev = to_dev(lay.tensors), to_dev(lay.items)
        self.hyper = torch.zeros(ngroups, 5, device=DEV)
        self.steps = torch.zeros(ngroups, dtype=torch.int32, device=DEV)
        self.sumsq = torch.zeros(1, device=DEV)
        self.gen = gen

    def args(self, gscale, max_norm, **over):
        lay = self.lay
        a = dict(p=self.p.data_ptr(), g=self.g.data_ptr(), codes=self.codes.data_ptr() if lay.code_bytes else None,
                 absmax=self.absmax.data_ptr() if lay.nblocks else None, state32=self.state32.data_ptr() if lay.small_numel else None,
                 maps=self.maps.data_ptr(), th=lay.tensors.ctypes.data, td=self.tensors_dev.data_ptr(), nt=len(lay.tensors),
                 ih=lay.items.ctypes.data, idv=self.items_dev.data_ptr(), ni=lay.items.size, n=self.n, cb=lay.code_bytes, nb=lay.nblocks,
                 sn=lay.small_numel, hyper=self.hyper.data_ptr(), steps=self.steps.data_ptr(), ng=self.ngroups, gs=gscale,
                 sumsq=self.sumsq.data_ptr(), mn=max_norm, st=stream_ptr())
        a.update(over)
        return list(a.values())

    def run(self, gscale, max_norm):
        call("hcp_adamw8bit_flat", *self.args(gscale, max_norm))

    def snapshot(self):
        return [t.cpu().numpy().copy() for t in (self.p, self.g, self.codes, self.absmax, self.state32)]


# four steps: per-group hyper rows (lr, beta1, beta2, eps, weight_decay), grad_scale, clip (None: max_norm 0; otherwise max_norm =
# clip x ||g grad_scale||, so < 1 engages it).  lr and beta1 are rewritten between steps, as OneCycleLR does; group 1 has wd 0.
def hyper_rows(k):
    lrs = [(1e-3, 5e-4, 2e-3), (5e-4, 1e-3, 1e-3), (2e-3, 1e-4, 5e-4), (1e-3, 1e-3, 1e-3)][k]
    b1 = [0.9, 0.85, 0.95, 0.9][k]
    return [(lrs[0], b1, 0.999, 1e-8, 1e-2), (lrs[1], b1, 0.99, 1e-6, 0.0), (lrs[2], 0.8, 0.999, 1e-8, 1e-1)]


A8_STEPS = [(0.5, 0.3), (1.0, 3.0), (0.5, None), (1.0, 0.5)]
NONFINITE_STEP = 2                                   # step 3 puts NaN / +inf / -inf into a few gradient elements

TABLES = {
    # 8-bit blocks of 1, 255, 256, 257 elements and tensors of several items (min_8bit_size 1: every tensor is 8-bit)
    "blocks8": ([1, 255, 256, 257, 511, 513, 64 * 256, 64 * 256 + 1, 3 * 64 * 256 + 17], 1),
    # tensors either side of min_8bit_size 4096, mixed modes and groups, small 32-bit tensors, a large 8-bit tensor
    "mixed": ([4095, 4096, 4097, 1, 255, 257, 300, 3 * 64 * 256 + 17, 1000003], 4096),
}


def fill_grads(tab, k, zero_block):
    """Gradient of step k: normal, a sixteenth exact zeros, and block 5 of the tensor `zero_block` all zero (with its scales 0 the
    block stays all-zero); at NONFINITE_STEP a few NaN / inf.  Returns the fp32 sum of squares of the finite elements."""
    g = torch.randn(tab.n + 16, generator=tab.gen, device=DEV) * (1 + k) * 1e-2
    g[torch.rand(tab.n + 16, generator=tab.gen, device=DEV) < 1 / 16] = 0.0
    if zero_block is not None:
        o = tab.offsets[zero_block]
        g[o + 5 * 256:o + 6 * 256] = 0.0
    if k == NONFINITE_STEP:
        for i, o in enumerate(tab.offsets):
            if tab.numels[i] > 8:
                g[o + 3], g[o + 5], g[o + tab.numels[i] - 1] = float("nan"), float("inf"), float("-inf")
    tab.g.copy_(g)
    fin = torch.isfinite(g)
    return float(torch.where(fin, g, 0).double().square().sum())


def check_step(tab, before, after, k, gs, stats):
    p0, g, c0, am0, st0 = before
    p1, _, c1, am1, st1 = after
    lay = tab.lay
    touched = np.zeros(tab.n + 16, dtype=bool)
    code_touched = np.zeros(c0.size, dtype=bool)
    for i, t in enumerate(lay.tensors):
        o, n, s = int(t["offset"]), int(t["numel"]), int(t["state"])
        hy = [float(h) for h in tab.hyper[int(t["group"])].cpu()]
        touched[o:o + n] = True
        if t["mode"] == 1:
            a, nb = int(t["absmax"]), -(-n // 256)
            pr, k1, k2, n1, n2, s1, s2 = R.step_8bit(p0[o:o + n], g[o:o + n], c0[s:s + n], c0[lay.code_bytes + s:lay.code_bytes + s + n],
                                                     am0[a:a + nb], am0[lay.nblocks + a:lay.nblocks + a + nb], hy, k + 1, gs)
            assert np.array_equal(am1[a:a + nb], n1) and np.array_equal(am1[lay.nblocks + a:lay.nblocks + a + nb], n2), f"tensor {i} absmax"
            blk = np.arange(n) // 256
            for got, want, s_, nm, code in ((c1[s:s + n], k1, s1, n1, R.MAP1), (c1[lay.code_bytes + s:lay.code_bytes + s + n], k2, s2, n2, R.MAP2)):
                with np.errstate(all="ignore"):
                    x = np.where(nm[blk] > 0, s_ / np.where(nm[blk] > 0, nm[blk], F32(1)), F32(0)).astype(F32)
                near = R.midpoint_distance(code, x) <= A8_TIE_ULPS
                bad = got != want
                stats["near"] += int(near.sum())
                stats["code_mismatch"] += int(bad.sum())
                assert not np.any(bad & ~near), f"tensor {i}: {int((bad & ~near).sum())} codes differ away from a midpoint"
            code_touched[s:s + n] = True
            code_touched[lay.code_bytes + s:lay.code_bytes + s + n] = True
            stats["zero_blocks"] += int((n1 == 0).sum())
        else:
            m, v = st0[s:s + n], st0[lay.small_numel + s:lay.small_numel + s + n]
            pr, mr, vr = R.step_32bit(p0[o:o + n], g[o:o + n], m, v, hy, k + 1, gs)
            for got, want, nm in ((st1[s:s + n], mr, "m"), (st1[lay.small_numel + s:lay.small_numel + s + n], vr, "v")):
                fin = np.isfinite(want)
                assert np.array_equal(np.isfinite(got), fin) and np.array_equal(np.isnan(got), np.isnan(want)), f"tensor {i} {nm} non-finite"
                err = np.abs(got[fin].astype(np.float64) - want[fin]) / (np.abs(want[fin].astype(np.float64)) + 1e-30)
                stats["m32"] = max(stats["m32"], float(err.max(initial=0.0)))
        got = p1[o:o + n]
        fin = np.isfinite(pr)
        assert np.array_equal(np.isnan(got), np.isnan(pr)) and np.array_equal(np.isfinite(got), fin), f"tensor {i} p non-finite"
        ref, base = pr[fin].astype(np.float64), p0[o:o + n][fin].astype(np.float64)
        # beyond one rounding of p', relative to the update; an element that must not move (update 0) may not differ at all
        upd = np.abs(ref - base)
        over = np.maximum(np.abs(got[fin] - ref) - np.spacing(np.abs(pr[fin])).astype(np.float64), 0.0)
        err = np.divide(over, upd, out=np.where(over > 0, np.inf, 0.0), where=upd > 0)
        stats["p_ulps"] = max(stats["p_ulps"], float((np.abs(got[fin] - ref) / np.spacing(np.abs(pr[fin])).astype(np.float64)).max(initial=0.0)))
        if err.size and float(err.max()) > stats["p"]:
            j = int(err.argmax())
            stats["p"] = float(err.max())
            stats["p_at"] = (i, int(t["mode"]), int(t["group"]), k + 1, float(base[j]), float(ref[j]), float(got[fin][j]), float(g[o:o + n][fin][j]))
        if t["mode"] == 1:                          # a non-finite gradient leaves p exactly
            nf = ~np.isfinite(g[o:o + n])
            assert np.array_equal(got[nf].view(np.int32), p0[o:o + n][nf].view(np.int32))
            stats["nonfinite8"] += int(nf.sum())
    assert np.array_equal(p1[~touched].view(np.int32), p0[~touched].view(np.int32)), "p written outside the tensors"
    assert np.array_equal(c1[~code_touched], c0[~code_touched]), "codes written outside the tensors"
    sm = lay.small_numel
    pad = np.ones(st0.size, dtype=bool)
    for t in lay.tensors[lay.tensors["mode"] == 0]:
        pad[int(t["state"]):int(t["state"]) + int(t["numel"])] = False
        pad[sm + int(t["state"]):sm + int(t["state"]) + int(t["numel"])] = False
    assert np.array_equal(st1[pad].view(np.int32), st0[pad].view(np.int32)), "state32 written outside the tensors"
    assert np.array_equal(am1[2 * lay.nblocks:].view(np.int32), am0[2 * lay.nblocks:].view(np.int32))


def run_table(name, check=True, seed=0, graph_step=None):
    numels, min8 = TABLES[name]
    tab = Table(numels, min8, seed=seed)
    zero_block = next((i for i, t in enumerate(tab.lay.tensors) if t["mode"] == 1 and t["numel"] > 6 * 256), None)
    if zero_block is not None:
        a = int(tab.lay.tensors[zero_block]["absmax"])
        tab.absmax[a + 5] = 0.0
        tab.absmax[tab.lay.nblocks + a + 5] = 0.0
    stats = {"near": 0, "code_mismatch": 0, "m32": 0.0, "p": 0.0, "p_ulps": 0.0, "zero_blocks": 0, "nonfinite8": 0}
    for k, (gscale, clip) in enumerate(A8_STEPS):
        ss = fill_grads(tab, k, zero_block)
        tab.hyper.copy_(torch.tensor(hyper_rows(k)))
        tab.sumsq.fill_(ss)
        ss32 = float(tab.sumsq)
        max_norm = 0.0 if clip is None else clip * math.sqrt(ss32) * gscale
        before = tab.snapshot() if check else None
        if graph_step == k:
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                tab.run(gscale, max_norm)
            gr.replay()
        else:
            tab.run(gscale, max_norm)
        assert tab.steps.tolist() == [k + 1] * tab.ngroups
        if check:
            gs = kernel_scale(gscale, ss32, max_norm)
            if clip is not None and clip < 1:
                assert gs < F32(gscale), "the clip must be engaged"
            check_step(tab, before, tab.snapshot(), k, gs, stats)
    return tab, stats


@pytest.mark.parametrize("name", list(TABLES))
def test_adamw8bit_flat_per_step(name):
    """Four steps of hcp_adamw8bit_flat over a table, each against the restatement from the kernel's own state: blocks of 1, 255,
    256, 257 elements, tensors either side of min_8bit_size, mixed modes and groups, offsets off multiples of 256, exact zeros and
    an all-zero block, non-finite gradients, the clip on and off, grad_scale 1/2, lr and beta1 rewritten between steps; nothing
    outside the tensors is written."""
    _, st = run_table(name)
    print(f"adamw8bit {name}: {st['near']} codes within {A8_TIE_ULPS} ulp of a midpoint, {st['code_mismatch']} codes differ, "
          f"{st['zero_blocks']} all-zero block scales, {st['nonfinite8']} non-finite 8-bit gradients")
    assert st["nonfinite8"] > 0
    if name == "mixed":
        assert st["zero_blocks"] >= len(A8_STEPS)
    measured(f"adamw8bit {name} m32/v32", st["m32"], A8_M32)
    print(f"adamw8bit {name}: worst |p' - p_ref| {st['p_ulps']:.1f} ulp; worst p (tensor, mode, group, step, p, p_ref, p', g): "
          f"{st.get('p_at')}")
    measured(f"adamw8bit {name} p", st["p"], A8_P)


def test_adamw8bit_flat_bit_identical_repeats_and_graph():
    """The same four steps twice give bit-identical buffers, and so does a run whose second step is a CUDA-graph replay."""
    runs = [run_table("mixed", check=False, seed=3), run_table("mixed", check=False, seed=3),
            run_table("mixed", check=False, seed=3, graph_step=1)]
    snaps = [tab.snapshot() for tab, _ in runs]
    for other in snaps[1:]:
        for a, b in zip(snaps[0], other):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_adamw8bit_refusals_before_launch_and_empty_table():
    """Null and misaligned pointers, bad sizes and bad table entries are refused before any launch (the step counters stay); an
    empty table launches nothing."""
    tab = Table([300, 5000, 8], 4096)
    tab.hyper.copy_(torch.tensor(hyper_rows(0)))
    before = _lib.launch_count
    snap = tab.snapshot()

    def rc(**over):
        r = _lib.lib().hcp_adamw8bit_flat(*tab.args(1.0, 0.0, **over))
        torch.cuda.synchronize()
        return r

    cases = [dict(p=None), dict(g=None), dict(codes=None), dict(absmax=None), dict(state32=None), dict(maps=None), dict(th=None),
             dict(td=None), dict(ih=None), dict(idv=None), dict(hyper=None), dict(steps=None),
             dict(p=tab.p.data_ptr() + 4), dict(g=tab.g.data_ptr() + 8), dict(codes=tab.codes.data_ptr() + 4),
             dict(state32=tab.state32.data_ptr() + 4), dict(absmax=tab.absmax.data_ptr() + 2),
             dict(n=-1), dict(ni=-1), dict(nt=-1), dict(cb=-16), dict(nb=-1), dict(sn=-4), dict(cb=tab.lay.code_bytes + 4),
             dict(sn=tab.lay.small_numel + 2), dict(ng=0), dict(ng=257), dict(ni=0),
             dict(n=tab.n - 12),                                # the last tensor reaches past p
             dict(cb=tab.lay.code_bytes - 16),                  # the 8-bit tensor's codes reach past code_bytes
             dict(nb=tab.lay.nblocks - 1),                      # ... and its scales past nblocks
             dict(sn=tab.lay.small_numel - 4),                  # a 32-bit tensor's m / v past small_numel
             dict(ng=2),                                        # tensor 2 is in group 2
             dict(ni=tab.lay.items.size - 1)]                   # the last tensor's blocks are not covered
    for over in cases:
        assert rc(**over) == HCP_ERR_INVALID, over
    bad_tables = []
    for field, value, row in (("offset", 2, 0), ("offset", 0, 1), ("numel", 0, 0), ("mode", 2, 0), ("group", -1, 0), ("state", 16, 1),
                              ("state", 2, 0), ("absmax", 1, 1)):
        t = tab.lay.tensors.copy()
        t[row][field] = value
        bad_tables.append(t)
    for t in bad_tables:
        assert rc(th=t.ctypes.data) == HCP_ERR_INVALID, t
    for fld, value, row in (("block0", 1, 0), ("block1", 1, 0), ("tensor", 2, 0), ("block1", 3, 0)):
        it = tab.lay.items.copy()
        it[row][fld] = value
        assert rc(ih=it.ctypes.data) == HCP_ERR_INVALID, (fld, value, row)
    assert rc(nt=0, th=None, td=None, ih=None, idv=None, ni=0) == 0
    assert _lib.launch_count == before
    assert tab.steps.tolist() == [0, 0, 0]
    for a, b in zip(snap, tab.snapshot()):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ----------------------------------------------------------------------------------------------------------------------------------
# the training step against the reference loop
# ----------------------------------------------------------------------------------------------------------------------------------
LR, WD = 1e-4, 1e-2
LORA_MIN8 = 512                 # TINY rank-4 factors (256 or 512 elements) are below 4096: this makes the 512-element ones 8-bit


def tiny_unet(sd, spec=U.TINY):
    u = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
                             cross_attention_dim=spec.cross_attention_dim)
    u.load_state_dict(sd)
    return u.to(DEV).requires_grad_(False).eval()


def copy_lora(group, lora):
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)


def cosine(name, got, want, bound):
    got, want = got.double(), want.double()
    cos = float(got @ want / (got.norm() * want.norm()))
    ratio = float(got.norm() / want.norm())
    measured(f"{name} update cosine", cos, bound, above=True)
    print(f"{name} update norm ratio {ratio:.4f}")
    assert 0.8 < ratio < 1.25


def lora_before(group):
    return {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in group.plugin_dict.items()}


def lora_delta(group, before, keys=None):
    return torch.cat([torch.cat([(group[k].layer.W_down - before[k][0]).flatten(), (group[k].layer.W_up - before[k][1]).flatten()]).cpu()
                      for k in (keys or group.plugin_dict)])


def ref_delta(lora, before, keys):
    return torch.cat([torch.cat([(lora[k][0].W_down.detach() - before[k][0].cpu()).flatten(),
                                 (lora[k][0].W_up.detach() - before[k][1].cpu()).flatten()]) for k in keys])


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("max_norm", [1e-3, 1e9])
def test_tiny_lora_adamw8bit_steps_match_reference_loop(use_graph, max_norm):
    """Three AdamW8bit steps of TINY attention LoRA, eager and graph replay, with a clip engaged at every step (1e-3) and never
    (1e9); min_8bit_size 512 puts the 512-element factors on the 8-bit path and leaves the 256-element ones on the 32-bit one."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, group = make_hcpdiff(unet, None, [{"lr": LR, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(group, lora)
    ref = R.use_adamw8bit(S.ReferenceLoop(sd, lora, spec, lr=LR, max_grad_norm=max_norm), weight_decay=WD, min_8bit_size=LORA_MIN8)
    before = lora_before(group)
    step = LoraTrainStep(unet, groups, lr=LR, weight_decay=WD, optimizer="adamw8bit", optimizer_kwargs={"min_8bit_size": LORA_MIN8},
                         max_grad_norm=max_norm, use_cuda_graph=use_graph)
    modes = step.a8_layout.tensors["mode"]
    assert 0 < int(modes.sum()) < modes.size
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=400 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    assert int(step.step_count) == 3 and step.a8_steps.tolist() == [3] * len(step.segments)
    cosine(f"lora graph={use_graph} max_norm={max_norm}", lora_delta(group, before), ref_delta(lora, before, list(group.plugin_dict)), COS)


def test_tiny_full_finetune_adamw8bit_steps_match_reference_loop():
    """Three AdamW8bit graph steps of every TINY UNet parameter (its convolution and attention weights 8-bit, its biases and norms
    32-bit), with EMA."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-5, "layers": [""]}], None)
    assert lora.empty() and len(groups) == 1
    names = [n for n, _ in unet.named_parameters()]
    ref_sd = {k: v.clone() for k, v in sd.items()}
    ref = R.use_adamw8bit(S.ReferenceLoop(ref_sd, None, spec, lr=1e-5, train_base=names), weight_decay=WD)
    p0 = {n: p.detach().clone() for n, p in unet.named_parameters()}
    step = LoraTrainStep(unet, groups, lr=1e-5, weight_decay=WD, optimizer="adamw8bit", ema={"decay_max": 0.999})
    modes = step.a8_layout.tensors["mode"]
    assert 0 < int(modes.sum()) < modes.size
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=300 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    du_p = torch.cat([(p.detach() - p0[n]).flatten().cpu() for n, p in unet.named_parameters()])
    du_r = torch.cat([(ref_sd[n].detach() - sd[n]).flatten() for n in names])
    cosine("full fine-tune", du_p, du_r, COS)
    ema = torch.cat([e.flatten() for e in step.ema_state().values()]).cpu()
    assert not torch.equal(ema, torch.cat([p0[n].flatten() for n in names]).cpu())
    assert step.optimizer_state_bytes < 4 * step.flat.numel                 # about 2 B per parameter against AdamW's 8


def test_joint_te_unet_adamw8bit_steps_match_reference_loop():
    """Three AdamW8bit steps of the TINY UNet + a two-layer text encoder, both adapter sets in their own groups, clip_skip 1 (the
    last layer's adapters get a zero gradient: their moments stay 0 and p only decays, as in the reference)."""
    spec, tspec = U.TINY, CR.TINY_TE
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(ugroup, lora)
    tsd = CR.init_params(tspec, seed=5)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=1e-5)
    tlora = CR.init_lora(tspec, rank=4)
    copy_lora(tgroup, tlora)
    opts = {"n_repeats": 1, "clip_skip": 1, "clip_final_norm": True}
    step = LoraTrainStep(unet, ugroups + tgroups, lr=1e-4, weight_decay=WD, optimizer="adamw8bit",
                         optimizer_kwargs={"min_8bit_size": LORA_MIN8}, text_encoder=te, text_encoder_opts=opts)
    ref = R.use_adamw8bit(CR.joint_reference_loop(sd, lora, spec, tsd, tlora, tspec, opts, lr=1e-4, te_lr=1e-5), weight_decay=WD,
                          min_8bit_size=LORA_MIN8)
    before_u, before_t = lora_before(ugroup), lora_before(tgroup)
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, spec, seed=100 + i)
        ids = CR.synthetic_ids(2, 1, seed=200 + i)
        loss = float(step.step(lat, noise, t, ids).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids)
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref), (i, loss, loss_ref)
    cosine("joint unet", lora_delta(ugroup, before_u), ref_delta(lora, before_u, list(ugroup.plugin_dict)), COS)
    live = [k for k in tgroup.plugin_dict if ".layers.1." not in k]
    cosine("joint te", lora_delta(tgroup, before_t, live), ref_delta(tlora, before_t, live), COS)
    skipped = [k for k in tgroup.plugin_dict if ".layers.1." in k]
    assert skipped
    for k in skipped:
        for got_p, ref_p, b0 in ((tgroup[k].layer.W_down, tlora[k][0].W_down, before_t[k][0]),
                                 (tgroup[k].layer.W_up, tlora[k][0].W_up, before_t[k][1])):
            assert not torch.equal(got_p, b0), f"{k}: not decayed"
            torch.testing.assert_close(got_p.detach().cpu(), ref_p.detach(), rtol=0, atol=float(np.spacing(np.float32(1.0))), msg=k)


def test_train_ac_ft_adamw8bit_yaml_tiny_xl_saves_and_resumes(tmp_path):
    """The entrypoint on cfgs/train/ft_adamw8bit_sdxl_synthetic.yaml with a TINY SDXL-shaped UNet: trains with a finite loss, saves
    the full UNet and resumes from it."""
    import yaml
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    with open(os.path.join(ROOT, "cfgs", "train", "ft_adamw8bit_sdxl_synthetic.yaml")) as f:
        cfg = yaml.safe_load(f)
    spec = U.TINY_XL
    cfg["model"]["unet"].update(sample_size=spec.sample_size, block_out_channels=list(spec.block_out_channels),
                                attention_head_dim=list(spec.num_heads), cross_attention_dim=spec.cross_attention_dim,
                                transformer_layers_per_block=list(spec.transformer_depth),
                                addition_time_embed_dim=spec.addition_time_embed_dim,
                                projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)
    cfg["exp_dir"] = str(tmp_path / "exp")
    cfg["train"].update(train_steps=3, save_step=3, log_step=1)
    cfg["data"].update(batch_size=2, num_samples=4)
    path = tmp_path / "ft_adamw8bit_tiny_xl.yaml"
    path.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", str(path)], cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    last = [ln for ln in r.stdout.splitlines() if ln.startswith("step 3/3")]
    assert last and math.isfinite(float(last[0].split("loss")[1].split()[0])), r.stdout
    ck = str(tmp_path / "exp" / "ckpts" / "unet-3.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert "base" in sd
    conf = load_config_with_cli(str(path), [f"train.resume.ckpt_path.unet=[{ck}]", "train.resume.start_step=3", "train.train_steps=4"])
    tr = Trainer(conf)
    assert tr.step_fn.optimizer == "adamw8bit" and tr.step_fn.betas == (0.9, 0.999)
    assert float(tr.step_fn.segments[0]["hyper"][4]) == pytest.approx(1e-3)
    assert int(tr.step_fn.a8_layout.tensors["mode"].sum()) > 0
    live = dict(tr.unet.named_parameters())
    for k, v in sd["base"].items():
        torch.testing.assert_close(live[k].detach().cpu(), v, msg=k, rtol=0, atol=0)
    tr.train()
