"""GPU tests of data groups (the reference's dict of datasets with per-group `loss_weight`, e.g. DreamBooth's prior-preservation
class set) and per-pixel loss masks (`att_mask`): the grouped masked loss kernel against fp64 torch, `LoraTrainStep.step_groups`
against the reference loop restated here (hcpdiff/train_ac.py:467-482: one forward / backward per group, gradient
sum_g loss_weight_g * loss_g, one clip and one optimizer step; get_loss :506-515 = (criterion * mask).mean()), and the entry point.

Tolerances as tests/test_gpu_step.py and tests/test_gpu_fullft.py: kernel per-group loss 2e-5 relative and dpred rel-L2 1e-5;
bf16 step vs fp32 oracle loss 2e-2, gradients rel-L2 5e-2, update cosine >= 0.9.  One concatenated UNet pass against the same
product run as one pass per group: rel-L2 1e-2 (the same bf16 arithmetic per sample, reductions over a different batch)."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import clip_ref as R

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import HcpError, call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {-1: None, 0: "MinSNRLoss", 1: "SoftMinSNRLoss", 2: "KDiffMinSNRLoss", 3: "EDMLoss"}


def rel_l2(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def cosine(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


# ----------------------------------------------------------------------------------------------------------------------
# the kernel
# ----------------------------------------------------------------------------------------------------------------------
def run_kernel(pred, target, t, mask, groups, weights, mode, gamma, grad_scale=1.0, dpred=True):
    B, C = pred.shape[:2]
    HW = pred[0, 0].numel()
    G = len(weights)
    sizes = [groups.count(g) for g in range(G)]
    scale = torch.tensor([weights[g] / (sizes[g] * C * HW) for g in groups], dtype=torch.float32, device=DEV)
    grp = torch.tensor(groups, dtype=torch.int32, device=DEV)
    acp = U.ddpm_alphas_cumprod().to(DEV)
    ws = torch.zeros((_lib.lib().hcp_eps_loss_grouped_workspace_bytes(B, C * HW) + 3) // 4, device=DEV)
    loss = torch.zeros(G, device=DEV)
    d = torch.full_like(pred, float("nan")) if dpred else None
    call("hcp_eps_loss_grouped", pred.data_ptr(), target.data_ptr(), t.data_ptr(), acp.data_ptr(), _lib.ptr(mask), scale.data_ptr(),
         grp.data_ptr(), G, mode, gamma, B, C, HW, grad_scale, loss.data_ptr(), _lib.ptr(d), ws.data_ptr(), ws.numel() * 4, stream_ptr())
    return loss, d


def fp64_reference(pred, target, t, mask, groups, weights, mode, gamma, grad_scale=1.0):
    B, C = pred.shape[:2]
    acp = U.ddpm_alphas_cumprod().double()
    p = pred.detach().double().cpu().requires_grad_(True)
    w = torch.ones(B, dtype=torch.float64) if mode < 0 else S.snr_weight(MODES[mode], gamma, t.cpu(), acp).double()
    m = torch.ones((B, 1) + tuple(pred.shape[2:]), dtype=torch.float64) if mask is None else mask.double().cpu().view(B, 1, *pred.shape[2:])
    per = (p - target.double().cpu()) ** 2 * w.view(-1, 1, 1, 1) * m
    losses = []
    for g in range(len(weights)):
        idx = [b for b in range(B) if groups[b] == g]
        losses.append(weights[g] * per[idx].mean())
    total = sum(losses)
    (total * grad_scale).backward()
    return torch.stack([x.detach() for x in losses]), p.grad


GROUPINGS = {1: [0], 3: [0, 1, 1], 5: [0, 0, 0, 1, 1]}


@pytest.mark.parametrize("HW", [63, 64, 4096, 16384])
@pytest.mark.parametrize("B", [1, 3, 5])
def test_grouped_loss_kernel_matches_fp64(golden_dir, B, HW):
    fx = torch.load(os.path.join(golden_dir, "ref_step.pt"))["loss"]
    gammas = sorted({float(k.split(":")[1]) for k in fx["out"]})
    groups = GROUPINGS[B]
    weights = [1.0, 0.5][:max(groups) + 1]
    g = torch.Generator().manual_seed(B * 100000 + HW)
    h = 7 if HW == 63 else int(math.isqrt(HW))
    shape = (B, 4, h, HW // h)
    pred, target = torch.randn(shape, generator=g).to(DEV), torch.randn(shape, generator=g).to(DEV)
    t = torch.randint(0, 1000, (B,), generator=g).to(DEV)
    masks = {"none": None, "random": (torch.rand((B, HW), generator=g) * 5).to(DEV), "zero": torch.zeros((B, HW), device=DEV)}
    for mode in (-1, 0, 1, 2, 3):
        for gamma in ([1.0] if mode < 0 else gammas):
            for mname, mask in masks.items():
                loss, d = run_kernel(pred, target, t, mask, groups, weights, mode, gamma, grad_scale=0.5)
                key = (mode, gamma, mname)
                if mname == "zero":
                    assert float(loss.abs().sum()) == 0.0 and float(d.abs().sum()) == 0.0, key
                    continue
                want, dwant = fp64_reference(pred, target, t, mask, groups, weights, mode, gamma, grad_scale=0.5)
                assert torch.all((loss.double().cpu() - want).abs() <= 2e-5 * want.abs()), (key, loss, want)
                assert rel_l2(d, dwant) <= 1e-5, key
                if mname == "none":               # NULL mask == ones mask, bit for bit; a repeat gives the same bits
                    l1, d1 = run_kernel(pred, target, t, torch.ones((B, HW), device=DEV), groups, weights, mode, gamma, grad_scale=0.5)
                    l2, _ = run_kernel(pred, target, t, None, groups, weights, mode, gamma, grad_scale=0.5)
                    assert torch.equal(loss, l1) and torch.equal(d, d1) and torch.equal(loss, l2), key


def test_grouped_loss_kernel_refuses_bad_arguments_before_launch():
    B, C, HW = 2, 4, 64
    x = torch.zeros((B, C, HW), device=DEV)
    t = torch.zeros(B, dtype=torch.int64, device=DEV)
    acp = U.ddpm_alphas_cumprod().to(DEV)
    scale, grp = torch.ones(B, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
    loss = torch.zeros(1, device=DEV)
    ws = torch.zeros(1024, device=DEV)
    good = dict(pred=x.data_ptr(), target=x.data_ptr(), t=t.data_ptr(), acp=acp.data_ptr(), mask=None, scale=scale.data_ptr(),
                group=grp.data_ptr(), G=1, mode=0, gamma=1.0, B=B, C=C, HW=HW, gs=1.0, loss=loss.data_ptr(), d=None, ws=ws.data_ptr(),
                wsb=ws.numel() * 4)
    bad = [dict(pred=None), dict(scale=None), dict(group=None), dict(loss=None), dict(ws=None), dict(mode=4), dict(mode=-2),
           dict(gamma=0.0), dict(t=None), dict(acp=None), dict(B=0), dict(C=0), dict(HW=0), dict(G=0), dict(B=70000), dict(wsb=0)]
    before = _lib.launch_count
    for change in bad:
        a = {**good, **change}
        with pytest.raises(HcpError):
            call("hcp_eps_loss_grouped", a["pred"], a["target"], a["t"], a["acp"], a["mask"], a["scale"], a["group"], a["G"], a["mode"],
                 a["gamma"], a["B"], a["C"], a["HW"], a["gs"], a["loss"], a["d"], a["ws"], a["wsb"], stream_ptr())
    assert _lib.launch_count == before
    # MSE needs neither t nor alphas_cumprod
    call("hcp_eps_loss_grouped", x.data_ptr(), x.data_ptr(), None, None, None, scale.data_ptr(), grp.data_ptr(), 1, -1, 0.0, B, C, HW, 1.0,
         loss.data_ptr(), None, ws.data_ptr(), ws.numel() * 4, stream_ptr())
    assert float(loss) == 0.0


# ----------------------------------------------------------------------------------------------------------------------
# the step
# ----------------------------------------------------------------------------------------------------------------------
def tiny_unet(sd, spec=U.TINY):
    down = tuple("CrossAttnDownBlock2D" if a else "DownBlock2D" for a in spec.down_has_attn)
    up = tuple("CrossAttnUpBlock2D" if a else "UpBlock2D" for a in spec.up_has_attn)
    u = UNet2DConditionModel(
        sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
        cross_attention_dim=spec.cross_attention_dim, down_block_types=down, up_block_types=up,
        transformer_layers_per_block=spec.transformer_depth, use_linear_projection=spec.use_linear_projection,
        addition_embed_type="text_time" if spec.addition_time_embed_dim else None, addition_time_embed_dim=spec.addition_time_embed_dim,
        projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)
    u.load_state_dict(sd)
    return u.to(DEV).requires_grad_(False).eval()


def lora_unet(spec, sd, rank=4):
    unet = tiny_unet(sd, spec)
    groups, group = make_hcpdiff(unet, None, [{"rank": rank, "alpha": 1.0, "dropout": 0.0, "lr": 1e-3, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=rank)
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)
    return unet, groups, group, lora


def group_batches(spec, sizes, it, masked=(0,), cfg=False, added=False):
    out = []
    for g, B in enumerate(sizes):
        lat, noise, t, ehs = U.synthetic_batch(B, spec, seed=1000 * it + 10 * g + 1)
        if cfg:
            ehs = torch.cat([U.synthetic_batch(B, spec, seed=1000 * it + 10 * g + 2)[3], ehs], 0)
        b = {"latents": lat, "noise": noise, "t": t, "ehs": ehs}
        if g in masked:
            b["mask"] = torch.rand((B, spec.sample_size, spec.sample_size), generator=torch.Generator().manual_seed(it * 7 + g)) * 5
        if added:
            b["added_cond_kwargs"] = U.synthetic_added_cond(B, spec, seed=1000 * it + 10 * g + 3)
        out.append(b)
    return out


class GroupedReference:
    """hcpdiff/train_ac.py:467-482 on the fp32 oracle: per group add_noise -> UNet -> (mse(reduction='none') * mask).mean() *
    loss_weight -> backward(/ accum); on the last micro-step clip_grad_norm_, AdamW, zero_grad."""

    def __init__(self, sd, lora, spec, weights, lr, accum=1, train_base=()):
        self.sd, self.lora, self.spec, self.weights, self.accum = sd, lora, spec, weights, accum
        self.acp = U.ddpm_alphas_cumprod()
        self.leaves = [sd[n].requires_grad_(True) for n in train_base]
        for blocks in (lora or {}).values():
            for e in blocks:
                self.leaves += [e.W_down.requires_grad_(True), e.W_up.requires_grad_(True)]
        self.opt = torch.optim.AdamW(self.leaves, lr=lr, weight_decay=1e-2)
        self.micro = 0

    def backward(self, batches):
        losses = []
        for b, w in zip(batches, self.weights):
            x_t = U.add_noise(b["latents"], b["noise"], b["t"], self.acp)
            pred = U.unet_forward(self.sd, x_t, b["t"], b["ehs"], lora=self.lora, spec=self.spec, added_cond_kwargs=b.get("added_cond_kwargs"))
            m = b.get("mask")
            m = torch.ones_like(pred[:, :1]) if m is None else m.view(pred.shape[0], 1, *pred.shape[2:])
            loss = (F.mse_loss(pred, b["noise"], reduction="none") * m).mean() * w
            (loss / self.accum).backward()
            losses.append(float(loss.detach()))
        return losses

    def micro_step(self, batches):
        losses = self.backward(batches)
        self.micro += 1
        if self.micro == self.accum:
            self.micro = 0
            torch.nn.utils.clip_grad_norm_(self.leaves, 1.0)
            self.opt.step()
            self.opt.zero_grad(set_to_none=False)
        return losses


@pytest.mark.parametrize("use_graph,accum", [(False, 1), (True, 1), (True, 2)])
def test_tiny_lora_groups_match_reference_loop(use_graph, accum):
    spec, sizes, weights = U.TINY, (2, 1), (1.0, 0.5)
    sd = U.init_params(spec)
    unet, groups, group, lora = lora_unet(spec, sd)
    p0 = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in group.plugin_dict.items()}
    ref = GroupedReference(sd, lora, spec, weights, lr=1e-3, accum=accum)
    step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=use_graph, grad_accum_steps=accum, loss_weights=weights)
    worst, moment_err = 0.0, None
    for it in range(3 * accum):
        batches = group_batches(spec, sizes, it)
        want = ref.micro_step(batches)
        got = step.step_groups(batches).cpu().tolist()
        worst = max(worst, max(abs(a - b) / abs(b) for a, b in zip(got, want)))
        if it == accum - 1:             # first moments after the first optimizer step = (1 - beta1) * clip * grad
            off = {id(p): o for p, o in zip(step.flat.params, step.flat.offsets)}
            num = den = 0.0
            for layer, blocks in lora.items():
                for prm, leaf in ((group[layer].layer.W_down, blocks[0].W_down), (group[layer].layer.W_up, blocks[0].W_up)):
                    m = step.m[off[id(prm)]:off[id(prm)] + prm.numel()].cpu().double()
                    mr = ref.opt.state[leaf]["exp_avg"].double().flatten()
                    num += float((m - mr).pow(2).sum())
                    den += float(mr.pow(2).sum())
            moment_err = math.sqrt(num / den)
    du_p = torch.cat([torch.cat([(b.layer.W_down - p0[k][0]).flatten(), (b.layer.W_up - p0[k][1]).flatten()]).detach().cpu()
                      for k, b in group.plugin_dict.items()])
    du_r = torch.cat([torch.cat([(lora[k][0].W_down.detach() - p0[k][0].cpu()).flatten(), (lora[k][0].W_up.detach() - p0[k][1].cpu()).flatten()])
                      for k in group.plugin_dict])
    print(f"[groups graph={use_graph} accum={accum}] loss {worst:.2e} moment {moment_err:.2e} cos {cosine(du_p, du_r):.4f}")
    assert worst < 2e-2 and moment_err < 5e-2
    assert cosine(du_p, du_r) > 0.9 and 0.9 < float(du_p.norm() / du_r.norm()) < 1.1


def test_tiny_full_finetune_groups_every_gradient_matches_oracle():
    spec, sizes, weights = U.TINY, (2, 1), (1.0, 0.5)
    sd = U.init_params(spec)
    unet = tiny_unet(sd, spec)
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-5, "layers": [""]}], None)
    step = LoraTrainStep(unet, groups, lr=1e-5, use_cuda_graph=False, grad_accum_steps=2, loss_weights=weights)
    batches = group_batches(spec, sizes, 0)
    got = step.step_groups(batches).cpu().tolist()              # first of two micro-steps: the gradient stays, scaled by 1/2
    torch.cuda.synchronize()
    ref_sd = {k: v.clone() for k, v in sd.items()}
    names = [n for n, _ in unet.named_parameters()]
    ref = GroupedReference(ref_sd, None, spec, weights, lr=1e-5, accum=2, train_base=names)
    want = ref.backward(batches)
    assert all(abs(a - b) < 2e-2 * abs(b) for a, b in zip(got, want)), (got, want)
    num = den = 0.0
    worst = []
    for name, p in unet.named_parameters():
        r = ref_sd[name].grad
        worst.append((rel_l2(p.grad, r), name))
        num += float((p.grad.cpu().double() - r.double()).pow(2).sum())
        den += float(r.double().pow(2).sum())
    worst.sort(reverse=True)
    print("global relL2", math.sqrt(num / den), "worst", worst[:4])
    assert math.sqrt(num / den) < 5e-2 and all(e < 0.25 for e, _ in worst)


def one_pass_vs_per_group(step, batches, weights):
    """flat gradient of ONE step_groups pass over every group vs the same engine run as one pass per group (the reference's
    loop, restated on the product): both inside one accumulation window of len(batches) + 1 micro-steps, so no optimizer runs."""
    step.loss_weights = list(weights)
    losses = step.step_groups(batches).cpu()
    one = step.flat.grad.clone()
    step.flat.grad.zero_()
    per = []
    for b, w in zip(batches, weights):
        step.loss_weights = [w]
        per.append(float(step.step_groups([b]).cpu()))
    two = step.flat.grad.clone()
    assert all(abs(a - b) <= 1e-2 * abs(b) for a, b in zip(losses.tolist(), per)), (losses, per)
    err = rel_l2(one, two)
    print(f"[one pass vs per group] grad rel {err:.2e}")
    assert float(two.norm()) > 0 and err <= 1e-2


def test_groups_with_text_encoder_match_per_group_passes():
    spec, tspec = U.TINY, R.TINY_TE
    sd = U.init_params(spec)
    unet, ugroups, _, _ = lora_unet(spec, sd)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(R.init_params(tspec, seed=5))
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=1e-5)
    tlora = R.init_lora(tspec, rank=4)
    with torch.no_grad():
        for layer, entries in tlora.items():
            tgroup[layer].layer.W_down.copy_(entries[0].W_down)
            tgroup[layer].layer.W_up.copy_(entries[0].W_up)
    step = LoraTrainStep(unet, ugroups + tgroups, use_cuda_graph=False, grad_accum_steps=4, text_encoder=te,
                         text_encoder_opts={"n_repeats": 1, "clip_skip": 0, "clip_final_norm": True})
    batches = group_batches(spec, (2, 1), 0)
    for g, b in enumerate(batches):
        b["ehs"] = R.synthetic_ids(b["latents"].shape[0], 1, seed=50 + g)
    one_pass_vs_per_group(step, batches, (1.0, 0.5))


def test_groups_with_sdxl_time_ids_match_per_group_passes():
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet = tiny_unet(sd, spec)
    pat = r".*\.attn.?$|.*\.ff$"
    groups, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "dropout": 0.0, "layers": ["re:" + pat]}])
    lora = U.init_lora(spec, rank=4, seed=3, pattern=pat)
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)
    step = LoraTrainStep(unet, groups, use_cuda_graph=False, grad_accum_steps=4)
    one_pass_vs_per_group(step, group_batches(spec, (2, 1), 0, added=True), (1.0, 0.5))


def test_groups_with_cfg_scale_match_per_group_passes():
    spec = U.TINY
    sd = U.init_params(spec)
    unet, groups, _, _ = lora_unet(spec, sd)
    step = LoraTrainStep(unet, groups, use_cuda_graph=False, grad_accum_steps=4, cfg_scale="1.0-3.0:cos")
    one_pass_vs_per_group(step, group_batches(spec, (2, 1), 0, cfg=True), (1.0, 0.5))


def test_one_group_without_mask_matches_step():
    """step() is step_groups() with one group of weight 1.  In the grouped run the last call is a step(): it replays the graphs
    step_groups() captured for that layout instead of capturing its own.  The first loss is computed from equal parameters and
    must be equal bit for bit; after that the LoRA weight gradients (summed with fp32 atomics) differ in their last bits between
    any two runs, the same path twice included, so parameters, moments and later losses are compared with tolerances."""
    spec = U.TINY
    results = []
    for grouped in (False, True):
        sd = U.init_params(spec)
        unet, groups, group, _ = lora_unet(spec, sd)
        step = LoraTrainStep(unet, groups, lr=1e-3, use_cuda_graph=True)
        losses = []
        for it in range(3):
            lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=500 + it)
            if grouped and it < 2:
                losses.append(step.step_groups([{"latents": lat, "noise": noise, "t": t, "ehs": ehs}]).cpu())
                graph = step._graph_fb
            else:
                losses.append(step.step(lat, noise, t, ehs).cpu())
        if grouped:
            assert step._graph_fb is graph
        results.append((torch.cat(losses), step.flat.data.clone(), step.m.clone()))
    (l0, p0, m0), (l1, p1, m1) = results
    assert torch.equal(l0[0], l1[0]) and torch.allclose(l0, l1, rtol=1e-4, atol=0), (l0, l1)
    assert rel_l2(p1, p0) <= 1e-4 and rel_l2(m1, m0) <= 1e-3


def test_step_groups_refusals_and_layout_check():
    spec = U.TINY
    sd = U.init_params(spec)
    unet, groups, _, _ = lora_unet(spec, sd)
    step = LoraTrainStep(unet, groups, use_cuda_graph=True, loss_weights=(1.0, 0.5))
    ok = group_batches(spec, (2, 1), 0)
    with pytest.raises(ValueError, match="loss_weights"):
        step.step_groups(ok[:1])
    small = dict(ok[1], latents=torch.randn(1, 4, 8, 8), noise=torch.randn(1, 4, 8, 8))
    with pytest.raises(ValueError, match="latent shape"):
        step.step_groups([ok[0], small])
    wide = dict(ok[1], ehs=torch.randn(1, 77, 32))
    with pytest.raises(ValueError, match="ehs"):
        step.step_groups([ok[0], wide])
    bad_mask = dict(ok[0], mask=torch.ones(2, 8, 8))
    with pytest.raises(ValueError, match="mask"):
        step.step_groups([bad_mask, ok[1]])
    assert step._static is None                                  # nothing was captured by the refused calls
    step.step_groups(ok)
    with pytest.raises(ValueError, match=re.escape("((2, 1), (1.0, 0.5), True)") + ".*" + re.escape("((2,), (1.0,), False)")):
        b = ok[0]
        step.step(b["latents"], b["noise"], b["t"], b["ehs"])


# ----------------------------------------------------------------------------------------------------------------------
# the entry point
# ----------------------------------------------------------------------------------------------------------------------
TINY_CFG = """
exp_dir: {exp}
seed: 7
model:
  unet:
    _target_: hcp_diffusion_b200.models.UNet2DConditionModel
    sample_size: 16
    block_out_channels: [64, 128, 128, 128]
    attention_head_dim: 2
    cross_attention_dim: 64
  init: random
lora_unet:
  - lr: 1.0e-3
    rank: 4
    layers: ['re:.*\\.attn.?$']
train:
  train_steps: 4
  save_step: 2
  log_step: 1
  scale_lr: true
  max_grad_norm: 1.0
  cuda_graph: true
  optimizer: {{lr: 1.0e-3, weight_decay: 1.0e-2}}
  scheduler: {{name: constant_with_warmup, num_warmup_steps: 1, num_training_steps: 4}}
data:
  dataset1:
    batch_size: 2
    path: {p1}
  dataset_class:
    batch_size: 1
    loss_weight: 0.5
    path: {p2}
"""


def test_train_ac_two_groups_from_files_saves_and_resumes(tmp_path):
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    g = torch.Generator().manual_seed(0)
    p1, p2 = os.path.join(tmp_path, "inst.pt"), os.path.join(tmp_path, "cls.pt")
    torch.save({"latents": torch.randn(6, 4, 16, 16, generator=g), "encoder_hidden_states": torch.randn(6, 77, 64, generator=g),
                "mask": torch.rand(6, 16, 16, generator=g) * 5}, p1)
    torch.save({"latents": torch.randn(4, 4, 16, 16, generator=g), "encoder_hidden_states": torch.randn(4, 77, 64, generator=g)}, p2)
    cfg_path = os.path.join(tmp_path, "groups.yaml")
    with open(cfg_path, "w") as f:
        f.write(TINY_CFG.format(exp=os.path.join(tmp_path, "exp"), p1=p1, p2=p2))
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", cfg_path, "train.train_steps=2"], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 2/2" in r.stdout
    ck = os.path.join(tmp_path, "exp", "ckpts", "unet-2.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert all(float(v.abs().sum()) > 0 for k, v in sd["lora"].items() if k.endswith("layer.W_up"))
    # the scheduler restarts on resume (its first warm-up step has lr 0), so train two more steps
    conf = load_config_with_cli(cfg_path, [f"train.resume.ckpt_path.unet=[{ck}]", "train.resume.start_step=2", "train.train_steps=4"])
    tr = Trainer(conf)
    assert [(n, bs, w) for n, _, bs, w in tr.groups] == [("dataset1", 2, 1.0), ("dataset_class", 1, 0.5)]
    assert tr.step_fn.loss_weights == [1.0, 0.5] and tr.sources[0]["mask"] is not None and tr.sources[1]["mask"] is None
    assert abs(tr.step_fn.segments[0]["base_lr"] - 3e-3) < 1e-12                  # scale_lr: (2 + 1) images
    live = tr.lora.state_dict()
    for k, v in sd["lora"].items():
        torch.testing.assert_close(live[k].cpu(), v, msg=k)
    before = {k: v.clone() for k, v in live.items()}
    tr.train()
    after = tr.lora.state_dict()
    assert any(not torch.equal(after[k], before[k]) for k in before if k.endswith("W_up"))
