"""Prodigy on the GPU (`pytest -m gpu`): hcp_prodigy_flat against a float64 run of tests/prodigy_ref.Prodigy, the training step with
optimizer='prodigy' against oracle.step_ref.ReferenceLoop running that restatement, and the entrypoint on a tiny copy of
cfgs/train/lora_prodigy_sd15_synthetic.yaml.

Kernel: several consecutive calls.  Before each call the restatement is loaded with the kernel's own state (p, p0, s, m, v as
fp32 values, and d, d_max, D_num, k from the fp64 block) and given the gradient the kernel sees, g * grad_scale_clip rounded to
fp32 as the kernel rounds it; it then runs one step in float64.  Errors, with u = 2^-24 and g~ = |g'| + |wd p| (the scale of the
gradient after coupled decay):
  m' within PD_STATE_ULP u of |beta1 m| + |d (1 - beta1)| g~;  v' of |beta2 v| + d^2 (1 - beta2) g~^2;  s' of |beta3 s| + |c_s| g~
  p' within PD_P_ULP u of |p| + |wd dlr p| + dlr m~ / (sqrt(v') + d eps), m~ the scale of m' above
  d and d_max within PD_D of the restatement's (relative), D_num within PD_D of |beta3 D_num| + (d / d0) dlr sum |g' (p0 - p)|.
Worst errors measured on one H100 80GB HBM3 (700 W): m' / v' / s' 3.27 u, p' 3.15 u, d 3.6e-8, D_num 5.4e-11.

Training step: Prodigy moves every parameter by about dlr along Adam's direction, so the update (after - before) of each model is
compared by its direction cosine and norm ratio, as test_gpu_lion.py does.
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

from hcp_diffusion_b200 import _lib, prodigy  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

import clip_ref as CR  # noqa: E402
import prodigy_ref as P  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HCP_ERR_INVALID = -1
F32 = np.float32
U24 = 2.0 ** -24

PD_STATE_ULP = 4.0              # m' / v' / s' in u of their scales
PD_P_ULP = 4.0                  # p' in u of its scale
PD_D = 1e-6                     # d, d_max, D_num relative
COS = 0.99                      # update cosine per model; measured 0.9995 / 0.9986 (LoRA, clip on / off), 0.9979 (full
                                # fine-tune), 0.9990 / 0.9988 (UNet / text-encoder adapters of the joint step)
D_RATIO = 1e-2                  # |d_engine / d_reference - 1| after three training steps; measured 9.1e-4


def measured(name: str, value: float, bound: float, above: bool = False) -> None:
    print(f"MEASURED {name}: {value:.6e} ({'>=' if above else '<='} {bound:.2e})")
    assert (value >= bound) if above else (value <= bound), f"{name}: {value:.6e} vs {bound:.2e}"


def gen(seed: int) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(seed)


def kernel_scale(gscale: float, sumsq: float, max_norm: float) -> np.float32:
    """gscale x clip as the kernel computes it in fp32 (af_grad_scale)."""
    gs, mn = F32(gscale), F32(max_norm)
    clip = F32(1.0)
    if mn > 0:
        norm = F32(np.sqrt(F32(sumsq))) * gs
        clip = min(F32(1.0), F32(mn / F32(norm + F32(1e-6))))
    return F32(gs * clip)


class Flat:
    """The kernel's buffers for segments [(count, lr, wd)]: each segment at a multiple of 4 after 8 sentinel elements, with 8
    sentinels between and after them; `check()`: nothing outside the segments was written."""

    SENTINEL = 12345.5

    def __init__(self, segs, opts, seed):
        self.segs, self.opts = segs, opts
        rows, off = [], 8
        for cnt, lr, wd in segs:
            rows.append((off, cnt, lr, wd))
            off += (cnt + 3) // 4 * 4 + 8
        self.n = off
        self.rows = rows
        g = gen(seed)
        self.buf = {k: torch.full((self.n,), self.SENTINEL, device=DEV) for k in ("p", "g", "p0", "s", "m", "v")}
        for off, cnt, _, _ in rows:
            self.buf["p"][off:off + cnt] = torch.randn(cnt, generator=g, device=DEV)
        self.table = prodigy.segment_table(rows)
        self.table_dev = torch.from_numpy(self.table.view(np.int64).reshape(len(rows), 4).copy()).to(DEV)
        self.hyper = torch.tensor(prodigy.hyper_row(opts, opts["betas"][0], opts["betas"][1], opts["eps"]), dtype=torch.float64, device=DEV)
        self.state = torch.tensor(prodigy.initial_state(opts["d0"]), dtype=torch.float64, device=DEV)
        self.work = torch.zeros(prodigy.WORKSPACE_BYTES // 8, dtype=torch.float64, device=DEV)
        self.step = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.sumsq = torch.zeros(1, device=DEV)

    def set_lrs(self, lrs):
        self.table_dev.view(torch.float64)[:, 2].copy_(torch.tensor(lrs, dtype=torch.float64))

    def seg(self, name, i):
        off, cnt, _, _ = self.rows[i]
        return self.buf[name][off:off + cnt]

    def run(self, gscale, max_norm):
        b = self.buf
        call("hcp_prodigy_flat", b["p"].data_ptr(), b["g"].data_ptr(), b["p0"].data_ptr(), b["s"].data_ptr(), b["m"].data_ptr(),
             b["v"].data_ptr(), self.n, self.table.ctypes.data, self.table_dev.data_ptr(), len(self.rows), self.hyper.data_ptr(),
             self.state.data_ptr(), self.work.data_ptr(), self.work.numel() * 8, gscale, self.sumsq.data_ptr(), max_norm,
             self.step.data_ptr(), stream_ptr())

    def check(self):
        inside = torch.zeros(self.n, dtype=torch.bool, device=DEV)
        for off, cnt, _, _ in self.rows:
            inside[off:off + cnt] = True
        for k, t in self.buf.items():
            if k != "g":
                assert bool((t[~inside] == self.SENTINEL).all()), f"{k}: written outside the segments"


def reference_step(fl: Flat, before, grads32, lrs):
    """One float64 restatement step from the kernel's state `before` ({name: [per-segment fp32 arrays]}, 'state': fp64 block)."""
    o = fl.opts
    ps = [torch.nn.Parameter(torch.from_numpy(x.astype(np.float64))) for x in before["p"]]
    groups = [{"params": [p], "lr": lr, "weight_decay": wd} for p, lr, (_, _, wd) in zip(ps, lrs, fl.segs)]
    opt = P.Prodigy(groups, lr=max(max(lrs), 1e-30), betas=o["betas"], beta3=o["beta3"], eps=o["eps"], decouple=o["decouple"],
                    use_bias_correction=o["use_bias_correction"], safeguard_warmup=o["safeguard_warmup"], d0=o["d0"], d_coef=o["d_coef"],
                    growth_rate=o["growth_rate"])
    st = before["state"]
    for g in opt.param_groups:
        g["d"], g["d_max"], g["d_numerator"], g["k"] = float(st[0]), float(st[1]), float(st[2]), int(st[3])
    if st[4]:
        for i, p in enumerate(ps):
            opt.state[p] = {"step": 0, **{k: torch.from_numpy(before[n][i].astype(np.float64))
                                           for k, n in (("s", "s"), ("p0", "p0"), ("exp_avg", "m"), ("exp_avg_sq", "v"))}}
    for p, g in zip(ps, grads32):
        p.grad = torch.from_numpy(g.astype(np.float64))
    opt.step()
    out = {"p": [p.detach().numpy() for p in ps], "s": [opt.state[p]["s"].numpy() for p in ps],
           "m": [opt.state[p]["exp_avg"].numpy() for p in ps], "v": [opt.state[p]["exp_avg_sq"].numpy() for p in ps]}
    g0 = opt.param_groups[0]
    out["scalars"] = (g0["d"], g0["d_max"], g0["d_numerator"], g0["k"])
    return out


def run_prodigy(segs, opts, steps, seed=0, check=True):
    """`steps`: [(gscale, clip (None: max_norm 0, else max_norm = clip x ||g gscale||), lr scale, zero gradient)].  Returns the
    worst errors {m, v, s, p, d, D_num} and the d trajectory."""
    fl = Flat(segs, opts, seed)
    g = gen(seed + 1)
    base = [torch.randn(cnt, generator=g, device=DEV) for cnt, _, _ in segs]    # a recurring component: the parameters travel
    zero = [torch.rand(cnt, generator=g, device=DEV) < 1 / 16 for cnt, _, _ in segs]
    worst = {k: 0.0 for k in ("m", "v", "s", "p", "d", "D_num")}
    ds, skipped = [], []
    for k, (gscale, clip, lr_scale, all_zero) in enumerate(steps):
        for i, (cnt, _, _) in enumerate(segs):
            gv = base[i] + 0.5 * torch.randn(cnt, generator=g, device=DEV)
            gv[zero[i]] = 0.0
            fl.seg("g", i).copy_(torch.zeros_like(gv) if all_zero else gv)
        lrs = [lr * lr_scale for _, lr, _ in segs]
        fl.set_lrs(lrs)
        ss = sum(float(fl.seg("g", i).double().square().sum()) for i in range(len(segs)))
        fl.sumsq.fill_(ss)
        max_norm = 0.0 if clip is None else clip * math.sqrt(ss) * gscale
        before = {n: [fl.seg(n, i).cpu().numpy().copy() for i in range(len(segs))] for n in ("p", "g", "p0", "s", "m", "v")}
        before["state"] = fl.state.cpu().numpy().copy()
        calls = int(fl.step)
        fl.run(gscale, max_norm)
        after = {n: [fl.seg(n, i).cpu().numpy() for i in range(len(segs))] for n in ("p", "p0", "s", "m", "v")}
        st = fl.state.cpu().numpy()
        assert int(fl.step) == calls + 1, "the EMA counter counts every call"
        gs = kernel_scale(gscale, ss, max_norm)
        if clip is not None and clip < 1 and ss > 0:
            assert gs < F32(gscale), "the clip must be engaged"
        grads32 = [(x * gs).astype(F32) for x in before["g"]]
        ref = reference_step(fl, before, grads32, lrs)
        skip = bool(st[5])
        skipped.append(skip)
        assert skip == (ref["scalars"][3] == int(before["state"][3])), "the kernel and the restatement disagree on skipping"
        assert st[4] == 1.0
        if skip:
            assert np.array_equal(st[[0, 1, 2, 3]], before["state"][[0, 1, 2, 3]]), "a skipped call keeps d, d_max, D_num, k"
            for i in range(len(segs)):
                assert np.array_equal(after["p"][i].view(np.int32), before["p"][i].view(np.int32)), "a skipped call keeps p"
        assert int(st[3]) == ref["scalars"][3]
        if not check:
            ds.append(float(st[0]))
            continue
        d_old, k_old = float(before["state"][0]), int(before["state"][3])
        o = opts
        b1, b2 = o["betas"]
        b3 = math.sqrt(b2) if o["beta3"] is None else o["beta3"]
        lr = max(lrs)
        bc = math.sqrt(1 - b2 ** (k_old + 1)) / (1 - b1 ** (k_old + 1)) if o["use_bias_correction"] else 1.0
        dlr = d_old * lr * bc
        cs = (d_old / o["d0"]) * (d_old if o["safeguard_warmup"] else dlr)
        d_new = float(st[0])
        dot_abs = 0.0
        for i, (cnt, lr_i, wd) in enumerate(segs):
            p0 = before["p"][i].astype(np.float64) if not before["state"][4] else before["p0"][i].astype(np.float64)
            pb = before["p"][i].astype(np.float64)
            wdc = 0.0 if o["decouple"] else wd
            gt = np.abs(grads32[i].astype(np.float64)) + np.abs(wdc * pb)
            if not before["state"][4]:
                assert np.array_equal(after["p0"][i].view(np.int32), before["p"][i].view(np.int32)), "p0 = p at the first call"
                mb = sb = vb = np.zeros(cnt)
            else:
                assert np.array_equal(after["p0"][i].view(np.int32), before["p0"][i].view(np.int32)), "p0 is written once"
                mb, sb, vb = (before[n][i].astype(np.float64) for n in ("m", "s", "v"))
            if lr_i * lr_scale > 0:
                dot_abs += float(np.sum(np.abs((grads32[i].astype(np.float64) + wdc * pb) * (p0 - pb))))
                scales = {"m": np.abs(b1 * mb) + d_old * (1 - b1) * gt, "v": np.abs(b2 * vb) + d_old ** 2 * (1 - b2) * gt ** 2,
                          "s": np.abs(b3 * sb) + abs(cs) * gt}
            else:
                scales = {n: np.zeros(cnt) for n in ("m", "v", "s")}
            for n in ("m", "v", "s"):
                err = np.abs(after[n][i].astype(np.float64) - ref[n][i])
                rel = np.divide(err, scales[n] * U24, out=np.where(err > 0, np.inf, 0.0), where=scales[n] > 0)
                worst[n] = max(worst[n], float(rel.max(initial=0.0)))
            if not skip:
                upd = dlr * scales["m"] / (np.sqrt(ref["v"][i]) + d_new * o["eps"])
                pscale = np.abs(pb) + abs((wd if o["decouple"] else 0.0) * dlr) * np.abs(pb) + upd
                err = np.abs(after["p"][i].astype(np.float64) - ref["p"][i])
                worst["p"] = max(worst["p"], float((err / (pscale * U24)).max(initial=0.0)))
        if not skip:
            for j, name in ((0, "d"), (1, "d")):
                worst[name] = max(worst[name], abs(float(st[j]) - ref["scalars"][j]) / ref["scalars"][j])
            dn_scale = abs(b3 * float(before["state"][2])) + (d_old / o["d0"]) * dlr * dot_abs
            if dn_scale > 0:
                worst["D_num"] = max(worst["D_num"], abs(float(st[2]) - ref["scalars"][2]) / dn_scale)
        ds.append(d_new)
    fl.check()
    return worst, ds, skipped, fl


def opts_of(**kw):
    return {**prodigy.check_options({}), **kw}


STEPS = [(1.0, None, 1.0, False), (0.5, 0.3, 1.0, False), (1.0, 3.0, 1.0, False), (0.5, None, 0.5, False), (1.0, 0.5, 1.0, False),
         (1.0, None, 1.0, False)]
# (name, segments [(count, lr, wd)], options)
CASES = [
    ("one element", [(1, 1.0, 0.0)], opts_of(d0=1e-3)),
    ("1-5 elements, lr-0 segment, decoupled", [(2, 1.0, 0.01), (3, 1.0, 0.0), (4, 0.0, 0.1), (5, 1.0, 0.01)], opts_of(d0=1e-3)),
    ("tails, coupled, bias correction", [(4099, 1.0, 0.01), (1026, 0.0, 0.05), (70001, 1.0, 0.0), (7, 1.0, 0.02)],
     opts_of(decouple=False, use_bias_correction=True, d0=1e-4)),
    ("safeguard warm-up, finite growth", [(4099, 1.0, 0.01), (1026, 0.0, 0.05), (70001, 1.0, 0.0)],
     opts_of(safeguard_warmup=True, growth_rate=1.02, d0=1e-4, betas=(0.95, 0.99), beta3=0.9)),
    ("grid-stride, all on", [((1 << 20) + 3, 1.0, 0.01), (9, 0.0, 0.5)],
     opts_of(use_bias_correction=True, safeguard_warmup=True, d0=1e-4, d_coef=0.5)),
]


@pytest.mark.parametrize("name,segs,opts", CASES, ids=[c[0] for c in CASES])
def test_prodigy_flat_consecutive_calls(name, segs, opts):
    """Six calls from the kernel's own state, each against the float64 restatement: tail-only segments, vector tails, several
    segments with an lr-0 one, coupled and decoupled decay, bias correction and safeguard warm-up on and off, a finite
    growth_rate, the clip engaged and not, grad_scale 1/2, the lr scaled down for one step."""
    worst, ds, skipped, _ = run_prodigy(segs, opts, STEPS)
    print(f"prodigy {name}: d over the calls {ds}")
    assert not any(skipped) and ds[-1] >= ds[0] == opts["d0"]
    for k in ("m", "v", "s"):
        measured(f"prodigy {name} {k}' ulps", worst[k], PD_STATE_ULP)
    measured(f"prodigy {name} p' ulps", worst["p"], PD_P_ULP)
    measured(f"prodigy {name} d relative", worst["d"], PD_D)
    measured(f"prodigy {name} D_num relative", worst["D_num"], PD_D)


def test_prodigy_flat_skipped_calls():
    """An all-zero gradient at the first call (D_den == 0), then a call at lr 0 (constant_with_warmup's first step): p, d,
    d_max, D_num and k stay, p0 is recorded at the first, the EMA counter advances on both; later calls run."""
    segs = [(4099, 1.0, 0.01), (6, 0.0, 0.1)]
    steps = [(1.0, None, 1.0, True), (1.0, None, 0.0, False), (1.0, 0.5, 1.0, False), (1.0, None, 1.0, False)]
    _, ds, skipped, fl = run_prodigy(segs, opts_of(d0=1e-3), steps)
    assert skipped == [True, True, False, False] and int(fl.step) == 4 and int(fl.state[3]) == 2


def test_prodigy_flat_graph_replays_bit_identical():
    """The three launches captured in one CUDA graph: replays from the same state are bit-identical, and equal eager calls."""
    segs = [((1 << 18) + 1, 1.0, 0.01), (1026, 0.0, 0.05), (4099, 1.0, 0.0)]
    opts = opts_of(use_bias_correction=True, d0=1e-4)
    results = []
    for mode in ("eager", "graph", "graph"):
        fl = Flat(segs, opts, seed=9)
        g = gen(10)
        fl.buf["g"].zero_()
        for i, (cnt, _, _) in enumerate(segs):
            fl.seg("g", i).copy_(torch.randn(cnt, generator=g, device=DEV))
        fl.sumsq.fill_(float(fl.buf["g"].double().square().sum()))
        if mode == "graph":                        # the eager run came first: the kernels are loaded before the capture
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                fl.run(0.5, 1.0)
            for _ in range(4):
                graph.replay()
        else:
            for _ in range(4):
                fl.run(0.5, 1.0)
        torch.cuda.synchronize()
        results.append([t.clone() for t in (fl.buf["p"], fl.buf["s"], fl.buf["m"], fl.buf["v"], fl.state)])
    print(f"d after four calls: {float(results[0][4][0]):.6e}")
    for other in results[1:]:
        for a, b in zip(results[0], other):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a.view(torch.int64),
                               b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int64))


def test_prodigy_refusals_before_launch_and_empty_table():
    """Null pointers, negative sizes, misaligned buffers, a short workspace and bad segments are refused before any launch (the
    state and counters stay); an empty table or one of empty segments is a no-op that launches nothing."""
    fl = Flat([(8, 1.0, 0.0), (8, 1.0, 0.0)], opts_of(), seed=3)
    b = fl.buf
    ptrs = [b[k].data_ptr() for k in ("p", "g", "p0", "s", "m", "v")]
    state0 = fl.state.clone()

    def rc(ptrs=ptrs, n=fl.n, table=fl.table, nsegs=2, hyper=None, state=None, work=None, wbytes=None, step=None):
        r = _lib.lib().hcp_prodigy_flat(*ptrs, n, None if table is None else table.ctypes.data, fl.table_dev.data_ptr(), nsegs,
                                        hyper or fl.hyper.data_ptr(), state or fl.state.data_ptr(), work or fl.work.data_ptr(),
                                        fl.work.numel() * 8 if wbytes is None else wbytes, 1.0, None, 0.0, step or fl.step.data_ptr(),
                                        stream_ptr())
        torch.cuda.synchronize()
        return r
    before = _lib.launch_count
    for j in range(6):
        bad = list(ptrs)
        bad[j] = None
        assert rc(ptrs=bad) == HCP_ERR_INVALID
        bad[j] = ptrs[j] + 4 * (j % 3 + 1)
        assert rc(ptrs=bad) == HCP_ERR_INVALID, j
    assert rc(table=None) == HCP_ERR_INVALID
    assert rc(n=-1) == HCP_ERR_INVALID and rc(nsegs=-1) == HCP_ERR_INVALID
    assert rc(wbytes=prodigy.WORKSPACE_BYTES - 8) == HCP_ERR_INVALID
    assert rc(state=fl.state.data_ptr() + 4) == HCP_ERR_INVALID and rc(work=fl.work.data_ptr() + 4) == HCP_ERR_INVALID
    for rows in ([(8, 8, 1.0, 0.0), (12, 8, 1.0, 0.0)],                  # overlapping
                 [(10, 8, 1.0, 0.0)],                                     # offset off 16-byte alignment
                 [(8, fl.n, 1.0, 0.0)],                                   # past n
                 [(8, -1, 1.0, 0.0)],                                     # negative count
                 [(24, 8, 1.0, 0.0), (8, 8, 1.0, 0.0)]):                  # decreasing
        assert rc(table=prodigy.segment_table(rows), nsegs=len(rows)) == HCP_ERR_INVALID, rows
    assert rc(nsegs=0) == 0
    assert rc(table=prodigy.segment_table([(8, 0, 1.0, 0.0)]), nsegs=1) == 0
    assert _lib.launch_count == before
    assert torch.equal(fl.state, state0) and int(fl.step) == 0
    assert bool((b["p0"] == Flat.SENTINEL).all()) and bool((b["m"] == Flat.SENTINEL).all())


# ----------------------------------------------------------------------------------------------------------------------------------
# the training step against the reference loop
# ----------------------------------------------------------------------------------------------------------------------------------
LR, WD, D0 = 1.0, 1e-2, 1e-4
PD_KW = {"d0": D0}


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


def d_agrees(name, step, ref):
    d, d_ref = float(step.pd_state[0]), ref.opt.param_groups[0]["d"]
    print(f"{name}: d {d:.6e}, reference {d_ref:.6e}")
    assert abs(d / d_ref - 1) < D_RATIO


def lora_delta(group, before):
    return torch.cat([torch.cat([(b.layer.W_down - before[k][0]).flatten(), (b.layer.W_up - before[k][1]).flatten()]).cpu()
                      for k, b in group.plugin_dict.items()])


def lora_before(group):
    return {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in group.plugin_dict.items()}


def ref_delta(group, lora, before):
    return torch.cat([torch.cat([(lora[k][0].W_down.detach() - before[k][0].cpu()).flatten(),
                                 (lora[k][0].W_up.detach() - before[k][1].cpu()).flatten()]) for k in group.plugin_dict])


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("max_norm", [1e-3, 1e9])
def test_tiny_lora_prodigy_steps_match_reference_loop(use_graph, max_norm):
    """Three Prodigy steps of TINY attention LoRA, eager and graph replay, with a clip engaged at every step (1e-3) and never (1e9)."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, group = make_hcpdiff(unet, None, [{"lr": LR, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(group, lora)
    ref = P.use_prodigy(S.ReferenceLoop(sd, lora, spec, lr=LR, max_grad_norm=max_norm), weight_decay=WD, **PD_KW)
    before = lora_before(group)
    step = LoraTrainStep(unet, groups, lr=LR, weight_decay=WD, optimizer="prodigy", optimizer_kwargs=PD_KW, max_grad_norm=max_norm,
                         use_cuda_graph=use_graph)
    assert step.optimizer_state_bytes == 16 * step.flat.numel
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=400 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    assert int(step.step_count) == 3 and int(step.pd_state[3]) == 3
    cosine(f"lora graph={use_graph} max_norm={max_norm}", lora_delta(group, before), ref_delta(group, lora, before), COS)
    d_agrees(f"lora graph={use_graph} max_norm={max_norm}", step, ref)


def test_tiny_full_finetune_prodigy_steps_match_reference_loop():
    """Three Prodigy graph steps of every TINY UNet parameter, with EMA."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, lora = make_hcpdiff(unet, [{"lr": LR, "layers": [""]}], None)
    assert lora.empty() and len(groups) == 1
    names = [n for n, _ in unet.named_parameters()]
    ref_sd = {k: v.clone() for k, v in sd.items()}
    ref = P.use_prodigy(S.ReferenceLoop(ref_sd, None, spec, lr=LR, train_base=names), weight_decay=WD, **PD_KW)
    p0 = {n: p.detach().clone() for n, p in unet.named_parameters()}
    step = LoraTrainStep(unet, groups, lr=LR, weight_decay=WD, optimizer="prodigy", optimizer_kwargs=PD_KW, ema={"decay_max": 0.999})
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=300 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    du_p = torch.cat([(p.detach() - p0[n]).flatten().cpu() for n, p in unet.named_parameters()])
    du_r = torch.cat([(ref_sd[n].detach() - sd[n]).flatten() for n in names])
    cosine("full fine-tune", du_p, du_r, COS)
    d_agrees("full fine-tune", step, ref)
    ema = torch.cat([e.flatten() for e in step.ema_state().values()]).cpu()
    assert int(step.step_count) == 3 and not torch.equal(ema, torch.cat([p0[n].flatten() for n in names]).cpu())


def test_joint_te_unet_prodigy_steps_match_reference_loop():
    """Three Prodigy steps of the TINY UNet + a two-layer text encoder, both adapter sets in their own groups at the same lr, one
    global d, clip_skip 1: the last layer's adapters get a zero gradient, so m = v = s = 0 and they only decay."""
    spec, tspec = U.TINY, CR.TINY_TE
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": LR, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(ugroup, lora)
    tsd = CR.init_params(tspec, seed=5)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [{"lr": LR, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=LR)
    tlora = CR.init_lora(tspec, rank=4)
    copy_lora(tgroup, tlora)
    opts = {"n_repeats": 1, "clip_skip": 1, "clip_final_norm": True}
    step = LoraTrainStep(unet, ugroups + tgroups, lr=LR, weight_decay=WD, optimizer="prodigy", optimizer_kwargs=PD_KW, text_encoder=te,
                         text_encoder_opts=opts)
    ref = P.use_prodigy(CR.joint_reference_loop(sd, lora, spec, tsd, tlora, tspec, opts, lr=LR, te_lr=LR), weight_decay=WD, **PD_KW)
    before_u, before_t = lora_before(ugroup), lora_before(tgroup)
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, spec, seed=100 + i)
        ids = CR.synthetic_ids(2, 1, seed=200 + i)
        loss = float(step.step(lat, noise, t, ids).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids)
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref), (i, loss, loss_ref)
    cosine("joint unet", lora_delta(ugroup, before_u), ref_delta(ugroup, lora, before_u), COS)
    d_agrees("joint", step, ref)
    live = [k for k in tgroup.plugin_dict if ".layers.1." not in k]
    skipped = [k for k in tgroup.plugin_dict if ".layers.1." in k]
    assert skipped

    def te_delta(keys, src):
        return torch.cat([torch.cat([(src(k)[0] - before_t[k][0].cpu()).flatten(), (src(k)[1] - before_t[k][1].cpu()).flatten()])
                          for k in keys])
    mine = lambda k: (tgroup[k].layer.W_down.detach().cpu(), tgroup[k].layer.W_up.detach().cpu())  # noqa: E731
    theirs = lambda k: (tlora[k][0].W_down.detach(), tlora[k][0].W_up.detach())                   # noqa: E731
    cosine("joint te", te_delta(live, mine), te_delta(live, theirs), COS)
    # the skipped layer's adapters only decay: p (1 - wd dlr) per step, the same direction as the reference's
    got, want = te_delta(skipped, mine), te_delta(skipped, theirs)
    assert bool(got.abs().gt(0).any())
    cosine("joint te skipped layer (decay only)", got, want, 0.9999)


def test_train_ac_lora_prodigy_yaml_tiny_saves_and_resumes(tmp_path):
    """The entrypoint on cfgs/train/lora_prodigy_sd15_synthetic.yaml with a TINY UNet: trains with a finite loss, saves the LoRA
    and resumes from it (the optimizer state is not checkpointed, as in the reference: Prodigy restarts from d0)."""
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    src = open(os.path.join(ROOT, "cfgs", "train", "lora_prodigy_sd15_synthetic.yaml")).read()
    exp = os.path.join(tmp_path, "exp")
    tiny = src.replace("exp_dir: exps/lora_prodigy_sd15_synthetic", f"exp_dir: {exp}").replace(
        "    _target_: hcp_diffusion_b200.models.UNet2DConditionModel\n",
        "    _target_: hcp_diffusion_b200.models.UNet2DConditionModel\n    sample_size: 16\n    block_out_channels: [64, 128, 128, 128]\n"
        "    attention_head_dim: 2\n    cross_attention_dim: 64\n")
    assert tiny != src
    cfg_path = os.path.join(tmp_path, "prodigy.yaml")
    with open(cfg_path, "w") as f:
        f.write(tiny)
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", cfg_path, "train.train_steps=3", "train.save_step=3",
                        "train.log_step=1", "data.batch_size=2", "data.num_samples=8"], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    last = [ln for ln in r.stdout.splitlines() if ln.startswith("step 3/3")]
    assert last and math.isfinite(float(last[0].split("loss")[1].split()[0])), r.stdout
    ck = os.path.join(exp, "ckpts", "unet-3.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    conf = load_config_with_cli(cfg_path, [f"train.resume.ckpt_path.unet=[{ck}]", "train.resume.start_step=3", "train.train_steps=4",
                                           "train.save_step=0", "data.batch_size=2", "data.num_samples=8"])
    tr = Trainer(conf)
    assert tr.step_fn.optimizer == "prodigy" and tr.step_fn.pd_hyper[7].item() == 7.0
    assert tr.step_fn.pd_segs_f64[:, 2:].tolist() == [[1.0, 0.01]]
    live = tr.lora.state_dict()
    for k, v in sd["lora"].items():
        torch.testing.assert_close(live[k].cpu(), v, msg=k, rtol=0, atol=0)
    before = {k: v.clone() for k, v in live.items()}
    tr.train()
    after = tr.lora.state_dict()
    assert any(not torch.equal(after[k], before[k]) for k in before if k.endswith("W_up"))
    assert int(tr.step_fn.pd_step) == 1
