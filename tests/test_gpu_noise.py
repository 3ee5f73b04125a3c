"""GPU tests of pyramid noise and zero-terminal-SNR schedules (`model.noise_scheduler`): hcp_pyramid_plan, hcp_pyramid_noise and
hcp_add_noise_scaled against the float64 restatement (tests/noise_ref.py) and against the reference PyramidNoiseScheduler's own
outputs (tests/golden/ref_noise.pt, made from the same draws), the engine under PyramidNoiseScheduler(ZeroTerminalScheduler(DDPM))
with MinSNRLoss against the reference loop assembled from the oracle pieces, and the entry point.

Bounds, from the first run on one H100 80GB HBM3 at a 700 W power limit (worst values printed by the tests):
  * plan: exact (level counts and sizes), 300 draws x 4 groups per shape.
  * pyramid target vs the float64 restatement: max |err| <= 5e-7 x max |target| (measured 1.9e-7; fp32 sums of up to 15 levels,
    torch's fp32 source index reproduced); vs the reference's own fp32 output the same bound.  1/std: 1.5e-7 relative (measured
    5.6e-8).  x_t: 5e-7 x max |x_t| (measured 1.8e-7).
  * steps: as tests/test_gpu_step.py (loss 2e-2 relative, update cosine >= 0.9, norm ratio in (0.9, 1.1)); measured loss 9.7e-4,
    cosine 0.995, norm ratio 0.9997 to 1.0002.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import noise_ref as N

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib, noise  # noqa: E402
from hcp_diffusion_b200._lib import HcpError, call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.ops import PyramidNoise  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402
from test_gpu_data_groups import cosine, group_batches, lora_unet  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TARGET_REL, STD_REL, XT_REL = 5e-7, 1.5e-7, 5e-7
DDPM = {"_target_": "diffusers.DDPMScheduler", "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear"}
PZ = {"_target_": "hcpdiff.noise.PyramidNoiseScheduler", "level": 10, "discount": 0.9, "step_size": 2.0,
      "base_scheduler": {"_target_": "hcpdiff.noise.ZeroTerminalScheduler", "base_scheduler": DDPM}}


def max_rel(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def run_pyramid(pn: PyramidNoise, base: torch.Tensor, sizes, plan=None):
    """(plan rows, target, inv_std) of one call; `plan`: an int32 [G, 32] plan written by the test instead of the plan kernel."""
    B, C, H, W = base.shape
    buf = pn.buffers(sizes, C, H, W)
    if plan is None:
        pn.plan(buf, H, W)
    else:
        buf["plan"].copy_(plan)
    target = torch.full_like(base, float("nan"))
    pn.pyramid(base, buf, target)
    torch.cuda.synchronize()
    return buf["plan"].cpu().clone(), target, buf["inv_std"].clone()


def plan_sizes(row):
    n = int(row[0])
    return [(int(row[2 + 2 * k]), int(row[3 + 2 * k])) for k in range(n)]


def restated(base, sizes_of_groups, starts, discount, seed, draw):
    out, inv = np.empty(base.shape, dtype=np.float64), []
    for g, sizes in enumerate(sizes_of_groups):
        t, s = N.pyramid(base[starts[g]:starts[g + 1]].cpu().numpy(), sizes, discount, seed, draw, g)
        out[starts[g]:starts[g + 1]] = t
        inv.append(s)
    return out, np.array(inv)


@pytest.mark.parametrize("step_size,H,W", [(2.0, 64, 64), (1.0, 128, 96), (3.0, 8, 8), (1.5, 96, 17)])
def test_plan_matches_restatement_exactly(step_size, H, W):
    pn = PyramidNoise(10, 0.9, step_size, DEV, seed=(1 << 36) + 5)
    buf = pn.buffers([1] * 4, 4, H, W)
    for draw in range(300):
        pn.plan(buf, H, W)
        rows = buf["plan"].cpu()
        for g in range(4):
            assert plan_sizes(rows[g]) == N.plan(pn.state[0].item(), draw, g, 10, step_size, H, W), (draw, g)
        pn.advance()
    assert int(pn.state[1]) == 300


def test_pyramid_matches_reference_golden(golden_dir):
    cases = torch.load(os.path.join(golden_dir, "ref_noise.pt"))["pyramid"]
    for c in cases:
        g, B = c["group"], c["B"]
        pn = PyramidNoise(c["level"], c["discount"], c["step_size"], DEV, seed=c["seed"])
        pn.state[1] = c["draw"]
        # the case's samples are data group g of the call: g one-sample groups come first
        base = torch.cat([torch.randn(g, 4, c["H"], c["W"]), N.golden_base_noise(c)]).to(DEV)
        plan, target, inv_std = run_pyramid(pn, base, [1] * g + [B])
        assert plan_sizes(plan[g]) == [tuple(s) for s in c["sizes"]]
        idx = c["index"].to(DEV)                            # the golden holds the reference's outputs at these flat indices
        e_t = max_rel(target[g:].flatten()[idx].cpu(), c["target"])
        e_s = abs(float(inv_std[g]) * c["std"] - 1.0)
        e_n = max_rel((target[g:] * inv_std[g]).flatten()[idx].cpu(), c["normalised"])
        print(f"[golden B={B} {c['H']}x{c['W']} level={c['level']} step={c['step_size']}] target {e_t:.2e} 1/std {e_s:.2e} normalised {e_n:.2e}")
        assert e_t <= TARGET_REL and e_s <= STD_REL and e_n <= TARGET_REL + STD_REL


@pytest.mark.parametrize("sizes,H,W,level,discount,step_size", [((2, 1, 3), 64, 64, 10, 0.9, 2.0), ((1,), 128, 128, 10, 0.9, 2.0),
                                                               ((4,), 96, 128, 6, 0.5, 1.0), ((1, 1), 8, 8, 3, 0.9, 3.0),
                                                               ((2, 2), 64, 64, 1, 0.9, 2.0)])
def test_pyramid_groups_match_restatement(sizes, H, W, level, discount, step_size):
    seed = 987654321
    pn = PyramidNoise(level, discount, step_size, DEV, seed=seed)
    gen = torch.Generator().manual_seed(sum(sizes) * 1000 + H)
    B = sum(sizes)
    base = torch.randn((B, 4, H, W), generator=gen).to(DEV)
    x0 = torch.randn((B, 4, H, W), generator=gen).to(DEV)
    t = torch.randint(0, 1000, (B,), generator=gen).to(DEV)
    t[0] = 999
    acp = noise.resolve(PZ).alphas_cumprod.to(DEV)
    starts = np.cumsum((0,) + tuple(sizes))
    for draw in range(3):
        x_t, target = pn.add_noise(x0, base, t, acp, sizes)
        torch.cuda.synchronize()
        buf = pn.buffers(sizes, 4, H, W)
        plans = [plan_sizes(r) for r in buf["plan"].cpu()]
        assert plans == [N.plan(seed, draw, g, level, step_size, H, W) for g in range(len(sizes))]
        want, inv = restated(base, plans, starts, discount, seed, draw)
        e_t = max_rel(target.cpu(), want)
        e_s = float(np.abs(buf["inv_std"].cpu().double().numpy() / inv - 1).max())
        a = acp.double().cpu()[t.cpu()].view(-1, 1, 1, 1).numpy()
        gi = np.repeat(np.arange(len(sizes)), sizes)
        xt_want = np.sqrt(a) * x0.double().cpu().numpy() + np.sqrt(1 - a) * want * inv[gi].reshape(-1, 1, 1, 1)
        e_x = max_rel(x_t.cpu(), xt_want)
        print(f"[groups {sizes} {H}x{W} level={level} step={step_size} draw={draw}] target {e_t:.2e} 1/std {e_s:.2e} x_t {e_x:.2e}")
        assert e_t <= TARGET_REL and e_s <= STD_REL and e_x <= XT_REL
        assert float(acp[999]) == 0.0 and torch.equal(x_t[0], target[0] * buf["inv_std"][0])     # x_t = noise at t = T-1
        if len(sizes) > 1:                       # each group draws its own grids and has its own std
            assert len(set(float(v) for v in buf["inv_std"].cpu())) == len(sizes)
        pn.advance()


def test_edge_plans_written_by_the_caller():
    H, W, B = 32, 24, 2
    pn = PyramidNoise(10, 0.9, 2.0, DEV, seed=3)
    base = torch.randn((B, 4, H, W)).to(DEV)
    rows = torch.zeros((1, 32), dtype=torch.int32)
    edges = [[], [(16, 12)], [(1, 12)], [(16, 1)], [(1, 1)], [(16, 12), (8, 6), (4, 3), (2, 1)]]
    for sizes in edges:
        rows.zero_()
        rows[0, 0] = len(sizes)
        for k, (h, w) in enumerate(sizes):
            rows[0, 2 + 2 * k], rows[0, 3 + 2 * k] = h, w
        _, target, inv = run_pyramid(pn, base, [B], plan=rows.to(DEV))
        want, winv = restated(base, [sizes], [0, B], 0.9, 3, 0)
        assert max_rel(target.cpu(), want) <= TARGET_REL and abs(float(inv[0]) / winv[0] - 1) <= STD_REL, sizes
    # sizes above the worst case of step_size and level counts above the cap are clamped to what the workspace holds
    rows.zero_()
    rows[0, 0], rows[0, 2], rows[0, 3] = 40, 1000, -5
    _, target, _ = run_pyramid(pn, base, [B], plan=rows.to(DEV))
    caps = [(16, 12), (8, 6), (4, 3), (2, 1)]
    got_sizes = [(min(max(int(rows[0, 2 + 2 * k]), 1), caps[k][0]), min(max(int(rows[0, 3 + 2 * k]), 1), caps[k][1])) for k in range(4)]
    want, _ = restated(base, [got_sizes], [0, B], 0.9, 3, 0)
    assert max_rel(target.cpu(), want) <= TARGET_REL


def test_bit_identical_on_repeat_and_in_a_graph_and_different_across_draws_and_seeds():
    H, W, sizes = 64, 64, (2, 1)
    x0, base = torch.randn((3, 4, H, W), device=DEV), torch.randn((3, 4, H, W), device=DEV)
    t = torch.tensor([0, 500, 999], device=DEV)
    acp = noise.resolve(PZ).alphas_cumprod.to(DEV)

    def eager(seed, draw):
        pn = PyramidNoise(10, 0.9, 2.0, DEV, seed=seed)
        pn.state[1] = draw
        x_t, target = pn.add_noise(x0, base, t, acp, sizes)
        return x_t.clone(), target.clone()

    a, b = eager(1, 0), eager(1, 0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(a[1], eager(1, 1)[1]) and not torch.equal(a[1], eager(2, 0)[1])
    pn = PyramidNoise(10, 0.9, 2.0, DEV, seed=1)
    pn.add_noise(x0, base, t, acp, sizes)                  # builds the layout's buffers outside the capture
    pn.state[1] = 0
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        x_t, target = pn.add_noise(x0, base, t, acp, sizes)
        pn.advance()
    got = []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        got.append((x_t.clone(), target.clone()))
    assert torch.equal(got[0][0], a[0]) and torch.equal(got[0][1], a[1])
    assert torch.equal(got[1][1], eager(1, 1)[1]) and torch.equal(got[2][0], eager(1, 2)[0])


def test_refusals_before_launch():
    B, C, H, W = 2, 4, 16, 16
    x = torch.zeros((B, C, H, W), device=DEV)
    state = torch.zeros(2, dtype=torch.int64, device=DEV)
    plan = torch.zeros((1, 32), dtype=torch.int32, device=DEV)
    gs = torch.tensor([0, B], dtype=torch.int32, device=DEV)
    inv = torch.zeros(1, device=DEV)
    t = torch.zeros(B, dtype=torch.int64, device=DEV)
    acp = torch.ones(1000, device=DEV)
    nbytes = _lib.lib().hcp_pyramid_workspace_bytes(B, C, H, W, 10, 2.0)
    assert nbytes > 0 and _lib.lib().hcp_pyramid_workspace_bytes(B, C, H, W, 10, 0.5) == 0
    ws = torch.zeros(nbytes // 4 + 8, device=DEV)
    good = dict(noise=x.data_ptr(), plan=plan.data_ptr(), gs=gs.data_ptr(), G=1, state=state.data_ptr(), level=10, discount=0.9, step=2.0,
                B=B, C=C, H=H, W=W, target=x.data_ptr(), inv=inv.data_ptr(), ws=ws.data_ptr(), wsb=nbytes)

    def pyr(a):
        call("hcp_pyramid_noise", a["noise"], a["plan"], a["gs"], a["G"], a["state"], a["level"], a["discount"], a["step"], a["B"], a["C"],
             a["H"], a["W"], a["target"], a["inv"], a["ws"], a["wsb"], stream_ptr())

    bad = [dict(noise=None), dict(plan=None), dict(gs=None), dict(state=None), dict(target=None), dict(inv=None), dict(ws=None),
           dict(noise=x.data_ptr() + 2), dict(target=x.data_ptr() + 1), dict(state=state.data_ptr() + 4), dict(ws=ws.data_ptr() + 4),
           dict(level=0), dict(level=17), dict(step=0.5), dict(step=float("nan")), dict(discount=float("inf")), dict(G=0), dict(G=65),
           dict(G=3), dict(B=-1), dict(C=0), dict(H=0), dict(W=0), dict(B=70000), dict(wsb=nbytes - 1)]
    before = _lib.launch_count
    for change in bad:
        with pytest.raises(HcpError):
            pyr({**good, **change})
    for args in ((None, 1, 10, 2.0, H, W, plan.data_ptr()), (state.data_ptr(), 1, 10, 2.0, H, W, None),
                 (state.data_ptr() + 4, 1, 10, 2.0, H, W, plan.data_ptr()), (state.data_ptr(), 0, 10, 2.0, H, W, plan.data_ptr()),
                 (state.data_ptr(), 1, 17, 2.0, H, W, plan.data_ptr()), (state.data_ptr(), 1, 10, 0.99, H, W, plan.data_ptr()),
                 (state.data_ptr(), 1, 10, 2.0, 0, W, plan.data_ptr())):
        with pytest.raises(HcpError):
            call("hcp_pyramid_plan", *args, stream_ptr())
    for args in ((None, x.data_ptr(), t.data_ptr(), acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 1, B, C * H * W, x.data_ptr()),
                 (x.data_ptr(), x.data_ptr(), t.data_ptr(), acp.data_ptr(), None, gs.data_ptr(), 1, B, C * H * W, x.data_ptr()),
                 (x.data_ptr() + 2, x.data_ptr(), t.data_ptr(), acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 1, B, C * H * W, x.data_ptr()),
                 (x.data_ptr(), x.data_ptr(), t.data_ptr() + 4, acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 1, B, C * H * W, x.data_ptr()),
                 (x.data_ptr(), x.data_ptr(), t.data_ptr(), acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 0, B, C * H * W, x.data_ptr()),
                 (x.data_ptr(), x.data_ptr(), t.data_ptr(), acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 1, -1, C * H * W, x.data_ptr())):
        with pytest.raises(HcpError):
            call("hcp_add_noise_scaled", *args, stream_ptr())
    assert _lib.launch_count == before
    pyr({**good, "B": 0})                                        # an empty batch is a no-op
    call("hcp_add_noise_scaled", x.data_ptr(), x.data_ptr(), t.data_ptr(), acp.data_ptr(), inv.data_ptr(), gs.data_ptr(), 1, 0, C * H * W,
         x.data_ptr(), stream_ptr())
    assert _lib.launch_count == before


# ----------------------------------------------------------------------------------------------------------------------
# the step: PyramidNoiseScheduler(ZeroTerminalScheduler(DDPMScheduler scaled_linear)) with MinSNRLoss(gamma 5)
# ----------------------------------------------------------------------------------------------------------------------
class PyramidReference:
    """hcpdiff/train_ac.py:437-482 on the fp32 oracle: per group make_noise with the pyramid (x_t from the normalised sum, the loss
    target the un-normalised one, both from the float64 restatement of the step's draws), UNet, (MinSNR * mask).mean() * weight,
    backward; clip_grad_norm_, AdamW, zero_grad."""

    def __init__(self, sd, lora, spec, sched, seed, weights, lr, kind="MinSNRLoss", gamma=5.0):
        self.sd, self.lora, self.spec, self.sched, self.seed, self.weights = sd, lora, spec, sched, seed, weights
        self.kind, self.gamma = kind, gamma
        self.acp = sched.alphas_cumprod
        self.leaves = []
        for blocks in lora.values():
            for e in blocks:
                self.leaves += [e.W_down.requires_grad_(True), e.W_up.requires_grad_(True)]
        self.opt = torch.optim.AdamW(self.leaves, lr=lr, weight_decay=1e-2)
        self.draw = 0

    def step(self, batches):
        p = self.sched.pyramid
        H, W = batches[0]["latents"].shape[2:]
        losses = []
        for g, (b, w) in enumerate(zip(batches, self.weights)):
            sizes = N.plan(self.seed, self.draw, g, p["level"], p["step_size"], H, W)
            target, inv = N.pyramid(b["noise"].numpy(), sizes, p["discount"], self.seed, self.draw, g)
            target = torch.from_numpy(target).float()
            x_t = U.add_noise(b["latents"], (target * inv).float(), b["t"], self.acp)
            pred = U.unet_forward(self.sd, x_t, b["t"], b["ehs"], lora=self.lora, spec=self.spec)
            m = b.get("mask")
            m = torch.ones_like(pred[:, :1]) if m is None else m.view(pred.shape[0], 1, *pred.shape[2:])
            per = F.mse_loss(pred, target, reduction="none") * S.snr_weight(self.kind, self.gamma, b["t"], self.acp).view(-1, 1, 1, 1)
            loss = (per * m).mean() * w
            loss.backward()
            losses.append(float(loss.detach()))
        self.draw += 1
        torch.nn.utils.clip_grad_norm_(self.leaves, 1.0)
        self.opt.step()
        self.opt.zero_grad(set_to_none=False)
        return losses


@pytest.mark.parametrize("use_graph,grouped", [(False, False), (True, False), (True, True)])
def test_tiny_lora_pyramid_ztsnr_min_snr_matches_reference_loop(use_graph, grouped):
    spec, seed = U.TINY, 4242
    sched = noise.resolve(PZ, {"type": "MinSNRLoss", "gamma": 5.0})
    sizes, weights = ((2, 1), (1.0, 0.5)) if grouped else ((3,), (1.0,))
    sd = U.init_params(spec)
    unet, groups, group, lora = lora_unet(spec, sd)
    p0 = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in group.plugin_dict.items()}
    ref = PyramidReference(sd, lora, spec, sched, seed, weights, lr=1e-3)
    step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=use_graph, loss={"type": "MinSNRLoss", "gamma": 5.0},
                         noise_scheduler=PZ, loss_weights=weights if grouped else None)
    step.set_noise_seed(seed)
    worst = 0.0
    for it in range(3):
        batches = group_batches(spec, sizes, it, masked=(0,) if grouped else ())
        batches[0]["t"][0] = 999                                    # zero terminal SNR: x_t = noise, MinSNR weight 1
        want = ref.step(batches)
        if grouped:
            got = step.step_groups(batches).cpu().tolist()
        else:
            b = batches[0]
            got = [float(step.step(b["latents"], b["noise"], b["t"], b["ehs"]).cpu())]
        worst = max(worst, max(abs(a - c) / abs(c) for a, c in zip(got, want)))
    assert int(step.pyramid.state[1]) == 3
    du_p = torch.cat([torch.cat([(b.layer.W_down - p0[k][0]).flatten(), (b.layer.W_up - p0[k][1]).flatten()]).detach().cpu()
                      for k, b in group.plugin_dict.items()])
    du_r = torch.cat([torch.cat([(lora[k][0].W_down.detach() - p0[k][0].cpu()).flatten(), (lora[k][0].W_up.detach() - p0[k][1].cpu()).flatten()])
                      for k in group.plugin_dict])
    ratio = float(du_p.norm() / du_r.norm())
    print(f"[pyramid graph={use_graph} groups={grouped}] loss {worst:.2e} cos {cosine(du_p, du_r):.4f} norm ratio {ratio:.4f}")
    assert worst < 2e-2 and cosine(du_p, du_r) > 0.9 and 0.9 < ratio < 1.1


def test_null_scheduler_step_is_unchanged_and_cfg_scale_runs():
    spec = U.TINY
    results = []
    for ns in (None, DDPM):                                 # an explicit SD1.x DDPM table is the default table, bit for bit
        sd = U.init_params(spec)
        unet, groups, _, _ = lora_unet(spec, sd)
        step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=True, noise_scheduler=ns)
        assert step.pyramid is None
        lat, nz, t, ehs = U.synthetic_batch(2, spec, seed=77)
        results.append((float(step.step(lat, nz, t, ehs).cpu()), step.flat.data.clone(), step.acp.clone()))
    # the same kernels on the same table
    assert torch.equal(results[0][2], results[1][2])
    assert abs(results[0][0] - results[1][0]) <= 1e-6 * abs(results[0][0])
    assert float((results[0][1] - results[1][1]).norm() / results[0][1].norm()) <= 1e-5
    sd = U.init_params(spec)
    unet, groups, _, _ = lora_unet(spec, sd)
    step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=True, cfg_scale="1.0-3.0:cos", noise_scheduler=PZ, loss="MinSNRLoss")
    for it in range(2):
        b = group_batches(spec, (2,), it, masked=(), cfg=True)[0]
        assert math.isfinite(float(step.step(b["latents"], b["noise"], b["t"], b["ehs"]).cpu()))
    with pytest.raises(ValueError, match="num_train_timesteps"):
        LoraTrainStep(unet, groups, noise_scheduler=PZ, num_train_timesteps=500)
    with pytest.raises(ValueError, match="EDMLoss"):
        LoraTrainStep(unet, groups, noise_scheduler=PZ, loss="EDMLoss")


def test_train_ac_pyramid_ztsnr_yaml_saves_and_resumes(tmp_path):
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    src = open(os.path.join(ROOT, "cfgs", "train", "lora_pyramid_ztsnr_sd15_synthetic.yaml")).read()
    exp = os.path.join(tmp_path, "exp")
    tiny = src.replace("exp_dir: exps/lora_pyramid_ztsnr_sd15_synthetic", f"exp_dir: {exp}").replace(
        "    _target_: hcp_diffusion_b200.models.UNet2DConditionModel\n",
        "    _target_: hcp_diffusion_b200.models.UNet2DConditionModel\n    sample_size: 16\n    block_out_channels: [64, 128, 128, 128]\n"
        "    attention_head_dim: 2\n    cross_attention_dim: 64\n")
    cfg_path = os.path.join(tmp_path, "pyr.yaml")
    with open(cfg_path, "w") as f:
        f.write(tiny)
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", cfg_path, "train.train_steps=2", "train.save_step=2",
                        "train.log_step=1", "data.batch_size=2", "data.num_samples=8"], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 2/2" in r.stdout
    ck = os.path.join(exp, "ckpts", "unet-2.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    conf = load_config_with_cli(cfg_path, [f"train.resume.ckpt_path.unet=[{ck}]", "train.resume.start_step=2", "train.train_steps=3",
                                           "train.save_step=0", "data.batch_size=2", "data.num_samples=8"])
    tr = Trainer(conf)
    assert tr.T == 1000 and tr.step_fn.pyramid is not None and float(tr.step_fn.acp[-1]) == 0.0
    live = tr.lora.state_dict()
    for k, v in sd["lora"].items():
        torch.testing.assert_close(live[k].cpu(), v, msg=k)
    before = {k: v.clone() for k, v in live.items()}
    tr.train()
    after = tr.lora.state_dict()
    assert any(not torch.equal(after[k], before[k]) for k in before if k.endswith("W_up"))
    assert int(tr.step_fn.pyramid.state[1]) == 1
