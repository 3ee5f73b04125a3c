"""GPU parity tests of the training step either side of the UNet call (`pytest -m gpu` on an H100).

Every kernel of `engine.LoraTrainStep` -- add_noise, the (SNR-weighted) loss and its gradient, the CFG mix, the global-norm
clip, AdamW, EMA -- against the fp32 oracle (oracle/step_ref.py, itself pinned to vectors of the real reference code in
tests/golden/ref_step.pt), then the whole step beside the reference loop (hcpdiff/train_ac.py:467-504 order:
forward -> loss -> backward -> clip_grad_norm_ -> torch.optim.AdamW -> zero_grad) on the TINY topology and at BASELINE
config 2 exactly (SD1.5, LoRA r=8 on the 128 attention linears, batch 4).

Tolerances: the flat fp32 kernels vs torch on EQUAL inputs: rel-L2 <= 1e-5 (loss / noise) and <= 1e-3 (parameters and Adam
moments after 5 steps); the full step (bf16 UNet vs fp32 oracle): loss per step within 2e-2, LoRA gradients / first moments
rel-L2 <= 5e-2, parameter UPDATE direction cosine >= 0.9 (Adam's m/sqrt(v) is +-1 at step 1: a 5 % gradient error only flips
the sign of near-zero entries).
"""
import ctypes as C
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib, ops  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def cosine(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def build(spec, sd, cfg_lora, lora_oracle):
    """Product UNet with the adapters of `cfg_lora` (reference yaml items) holding the oracle's LoRA values."""
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    groups, group = make_hcpdiff(unet, None, cfg_lora)
    with torch.no_grad():
        for layer, entries in lora_oracle.items():
            blk = group[layer]
            blk.layer.W_down.copy_(entries[0].W_down)
            blk.layer.W_up.copy_(entries[0].W_up)
    assert set(lora_oracle) == set(group.plugin_dict)
    return unet, groups, group


# ----------------------------------------------------------------------------------------------------------------------
# flat kernels vs torch / the pinned step oracle on equal inputs
# ----------------------------------------------------------------------------------------------------------------------
def test_add_noise_and_losses_match_oracle(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "ref_step.pt"))["loss"]
    acp = U.ddpm_alphas_cumprod()
    pred, target, t = fx["pred"].to(DEV), fx["target"].to(DEV), fx["t"].to(DEV)
    B, per = pred.shape[0], pred[0].numel()
    # add_noise (reference make_noise / DDPMScheduler.add_noise, train_ac.py:437-447)
    xt = torch.empty_like(pred)
    call("hcp_add_noise", pred.data_ptr(), target.data_ptr(), t.data_ptr(), acp.to(DEV).data_ptr(), B, per, xt.data_ptr(), stream_ptr())
    assert rel_l2(xt, U.add_noise(fx["pred"], fx["target"], fx["t"], acp)) < 1e-6
    # plain MSE (nn.MSELoss(reduction='none').mean()) incl. the accumulation scale on the gradient only
    p = fx["pred"].clone().requires_grad_(True)
    ref = S.eps_loss(p, fx["target"], fx["t"], acp)
    ref.backward()
    loss, dpred = torch.zeros(1, device=DEV), torch.empty_like(pred)
    call("hcp_mse_loss", pred.data_ptr(), target.data_ptr(), pred.numel(), 0.5, loss.data_ptr(), dpred.data_ptr(), stream_ptr())
    assert abs(float(loss) - float(ref)) < 1e-5 * float(ref) and rel_l2(dpred, 0.5 * p.grad) < 1e-5
    # the four SNR-weighted criteria against the REAL reference classes' outputs
    for key, want in fx["out"].items():
        kind, gamma = key.split(":")
        mode = {"MinSNRLoss": 0, "SoftMinSNRLoss": 1, "KDiffMinSNRLoss": 2, "EDMLoss": 3}[kind]
        loss.zero_()
        call("hcp_snr_mse_loss", pred.data_ptr(), target.data_ptr(), t.data_ptr(), acp.to(DEV).data_ptr(), float(gamma), mode, per, pred.numel(), 1.0,
             loss.data_ptr(), dpred.data_ptr(), stream_ptr())
        assert abs(float(loss) - float(want["loss"])) < 2e-5 * abs(float(want["loss"])), key
        assert rel_l2(dpred, want["dpred"]) < 2e-5, key


def test_cfg_mix_matches_reference_context(golden_dir):
    from hcp_diffusion_b200.engine import CFG_RATE_MODES, _CfgMixFn, get_cfg_range
    for c in torch.load(os.path.join(golden_dir, "ref_step.pt"))["cfg"]:
        lo, hi, fn = get_cfg_range(c["text"])
        assert (lo, hi, fn) == tuple(c["range"])
        eps2 = c["eps2"].to(DEV).requires_grad_(True)
        out = _CfgMixFn.apply(eps2, c["t"].to(DEV), lo, hi, CFG_RATE_MODES[fn], 1000)
        assert rel_l2(out, c["out"]) < 1e-6
        out.backward(c["dout"].to(DEV))
        assert rel_l2(eps2.grad, c["deps2"]) < 1e-6


@pytest.mark.parametrize("max_norm,grad_scale", [(1.0, 1.0), (1.0, 1e-3), (0.0, 1.0)])
def test_clip_adamw_ema_match_torch_on_equal_grads(max_norm, grad_scale):
    """hcp_sumsq + hcp_adamw_flat_dev (+ hcp_ema_flat) over two parameter groups vs clip_grad_norm_ + torch.optim.AdamW (+ the
    reference EMA rule) fed the SAME fp32 gradients for 5 steps; grad_scale 1e-3 makes the clip inactive."""
    g = torch.Generator().manual_seed(0)
    shapes = [(8, 320), (320, 8), (8, 768), (1280, 8), (7,)]
    ref_p = [torch.randn(s, generator=g).requires_grad_(True) for s in shapes]
    prod_p = [torch.nn.Parameter(p.detach().clone().to(DEV)) for p in ref_p]
    lrs = (1e-3, 4e-4)
    opt = torch.optim.AdamW([{"params": ref_p[:3], "lr": lrs[0]}, {"params": ref_p[3:], "lr": lrs[1]}], weight_decay=1e-2)
    step = LoraTrainStep(torch.nn.Identity(), [{"params": prod_p[:3], "lr": lrs[0]}, {"params": prod_p[3:], "lr": lrs[1]}], weight_decay=1e-2,
                         max_grad_norm=max_norm, use_cuda_graph=False, ema={"decay_max": 0.9997, "power": 0.85})
    ema_ref = [p.detach().clone() for p in ref_p]
    for it in range(1, 6):
        grads = [torch.randn(s, generator=g) * grad_scale * (1 + it) for s in shapes]
        for p, gr in zip(ref_p, grads):
            p.grad = gr.clone()
        for p, gr in zip(prod_p, grads):
            p.grad.copy_(gr)                       # the flat gradient buffer
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_(ref_p, max_norm)
        opt.step()
        ema_ref = [S.ema_update(e, p.detach(), it, decay_max=0.9997, power=0.85) for e, p in zip(ema_ref, ref_p)]
        step._optimizer()
        assert float(step.flat.grad.abs().sum()) == 0.0            # zero_grad after the step (train_ac.py:494)
    emas = step.ema_state()
    for i, (p, q) in enumerate(zip(prod_p, ref_p)):
        assert rel_l2(p, q) < 1e-3
        assert rel_l2(emas[p], ema_ref[i]) < 1e-3
    for q, (off, p) in zip(ref_p, zip(step.flat.offsets, prod_p)):
        n = q.numel()
        assert rel_l2(step.m[off:off + n], opt.state[q]["exp_avg"]) < 1e-3
        assert rel_l2(step.v[off:off + n], opt.state[q]["exp_avg_sq"]) < 1e-3
    assert [int(s["step"]) for s in step.segments] == [5, 5]


# ----------------------------------------------------------------------------------------------------------------------
# the whole step beside the reference loop
# ----------------------------------------------------------------------------------------------------------------------
def run_side_by_side(spec, batch, rank, steps, lr, use_graph, accum=1, loss=None, ema=None, two_groups=False, cfg_scale=None, ctx_len=77):
    sd = U.init_params(spec)
    lora = U.init_lora(spec, rank=rank)
    if two_groups:          # two `lora_unet:` items with their own lr (reference cfg_net_tools.py:107-127): attn1 layers / attn2 layers
        cfg = [{"rank": rank, "alpha": 1.0, "dropout": 0.0, "lr": lr, "layers": [r"re:.*\.attn1$"]},
               {"rank": rank, "alpha": 1.0, "dropout": 0.0, "lr": lr * 0.25, "layers": [r"re:.*\.attn2$"]}]
        group_of = lambda layer, bi, e: 0 if ".attn1." in layer else 1   # noqa: E731
        lrs = {0: lr, 1: lr * 0.25}
    else:
        cfg = [{"rank": rank, "alpha": 1.0, "dropout": 0.0, "lr": lr, "layers": [r"re:.*\.attn.?$"]}]
        group_of, lrs = None, None
    unet, groups, group = build(spec, sd, cfg, lora)
    p0 = {layer: (group[layer].layer.W_down.detach().clone(), group[layer].layer.W_up.detach().clone()) for layer in lora}
    kind, gamma = (None, 1.0) if loss is None else (loss["type"], loss["gamma"])
    cfg_range = None if cfg_scale is None else S.get_cfg_range(cfg_scale)
    ref = S.ReferenceLoop(sd, lora, spec, lr=lr, accum=accum, loss_kind=kind, gamma=gamma, ema_kw=ema, group_of=group_of, lrs=lrs,
                          cfg_scale=cfg_range)
    step = LoraTrainStep(unet, groups, lr=lr, use_cuda_graph=use_graph, grad_accum_steps=accum, loss=loss, ema=ema, cfg_scale=cfg_scale)
    worst = 0.0
    for it in range(steps * accum):
        lat, noise, t, ehs = U.synthetic_batch(batch, spec, seed=100 + it, ctx_len=ctx_len)
        if cfg_scale is not None:
            ehs = torch.cat([U.synthetic_batch(batch, spec, seed=900 + it, ctx_len=ctx_len)[3], ehs], 0)     # [negative | positive]
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        worst = max(worst, abs(l_prod - l_ref) / abs(l_ref))
        if it == accum - 1:
            # first optimizer step: gradients are gone (zero_grad) but the first moments are (1 - beta1) * clip * grad
            num = den = 0.0
            moms = ref.moments()
            offset_of = {id(p): o for p, o in zip(step.flat.params, step.flat.offsets)}
            i = 0
            for layer, blocks in lora.items():
                for e in blocks:
                    for prod_param, _ in ((group[layer].layer.W_down, 0), (group[layer].layer.W_up, 1)):
                        off = offset_of[id(prod_param)]
                        got = step.m[off:off + prod_param.numel()].view_as(prod_param)
                        num += float((got.cpu().double() - moms[i][0].double()).pow(2).sum())
                        den += float(moms[i][0].double().pow(2).sum())
                        i += 1
            first_moment_err = math.sqrt(num / den)
    du_prod, du_ref = [], []
    for layer, blocks in lora.items():
        for got, want, start in ((group[layer].layer.W_down, blocks[0].W_down, p0[layer][0]), (group[layer].layer.W_up, blocks[0].W_up, p0[layer][1])):
            du_prod.append((got.detach().cpu() - start.cpu()).flatten())
            du_ref.append((want.detach() - start.cpu()).flatten())
    du_prod, du_ref = torch.cat(du_prod), torch.cat(du_ref)
    out = {"loss_err": worst, "moment_err": first_moment_err, "update_cos": cosine(du_prod, du_ref),
           "update_norm_ratio": float(du_prod.norm() / du_ref.norm()), "step": step, "ref": ref, "lora": lora, "group": group}
    print({k: v for k, v in out.items() if isinstance(v, float)})
    return out


def check(out):
    assert out["loss_err"] < 2e-2
    assert out["moment_err"] < 5e-2
    assert out["update_cos"] > 0.9 and 0.9 < out["update_norm_ratio"] < 1.1


@pytest.mark.parametrize("use_graph", [False, True])
def test_tiny_train_step_matches_reference_loop(use_graph):
    check(run_side_by_side(U.TINY, batch=4, rank=4, steps=4, lr=1e-3, use_graph=use_graph))


def test_tiny_train_step_accumulation_two_groups_minsnr_ema():
    """gradient_accumulation_steps = 2, two parameter groups with different lr, MinSNRLoss(gamma 2) and EMA, all at once."""
    out = run_side_by_side(U.TINY, batch=2, rank=4, steps=3, lr=1e-3, use_graph=True, accum=2, loss={"type": "MinSNRLoss", "gamma": 2.0},
                           ema={"decay_max": 0.9997, "power": 0.85}, two_groups=True)
    check(out)
    step, ref = out["step"], out["ref"]
    assert [int(s["step"]) for s in step.segments] == [3, 3]
    # EMA of the product tracks the product's parameters with the reference rule; compare with the oracle's EMA the same way as the update
    emas = step.ema_state()
    num = den = 0.0
    i = 0
    for layer, blocks in out["lora"].items():
        for prm in (out["group"][layer].layer.W_down, out["group"][layer].layer.W_up):
            num += float((emas[prm].cpu().double() - ref.ema[i].double()).pow(2).sum())
            den += float(ref.ema[i].double().pow(2).sum())
            i += 1
    assert math.sqrt(num / den) < 1e-2


def test_tiny_dreamartist_cfg_step_matches_reference_loop():
    """DreamArtistPTContext training (cfg_scale '1.0-3.0:cos'): doubled batch [latents | latents] x [negative | positive] text."""
    check(run_side_by_side(U.TINY, batch=2, rank=4, steps=3, lr=1e-3, use_graph=True, cfg_scale="1.0-3.0:cos"))


def test_sd15_config2_train_step_matches_reference_loop():
    """BASELINE config 2 exactly: SD1.5, LoRA r=8 on every attn1/attn2 Linear, batch 4, 64x64 latents, 77 tokens; 3 steps beside the
    fp32 reference loop (the benchmark's own configuration, captured in CUDA graphs like bench.py runs it)."""
    check(run_side_by_side(U.SD15, batch=4, rank=8, steps=3, lr=1e-4, use_graph=True))
