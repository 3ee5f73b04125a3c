"""GPU tests of training LoRA on the text encoder together with the UNet (`pytest -m gpu`): the UNet's fp32 gradient for the text
embedding, the joint step against the reference loop (tests/clip_ref.joint_reference_loop: the text encoder, the UNet and one
AdamW over both adapter sets with a shared global-norm clip), and the entrypoint with `lora_text_encoder`.

Bounds (measured on one H100 80GB HBM3 at a 400 W power limit):
  d(ehs) of the TINY UNet vs the fp32 oracle, relative L2: measured 2.89e-2 (inline and hoisted k/v), bound 5e-2.
  Joint step, as tests/test_gpu_step.py: loss per step within 2e-2 relative (measured 7.7e-4), parameter update (after - before)
  per model: direction cosine >= 0.9 (measured >= 0.997) and norm ratio in (0.9, 1.1) (measured 0.9999-1.0009).
"""
import os
import subprocess
import sys

import pytest
import torch

import clip_ref as R

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib, ops  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def tiny_unet(sd, spec=U.TINY):
    u = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
                             cross_attention_dim=spec.cross_attention_dim)
    u.load_state_dict(sd)
    return u.to(DEV).requires_grad_(False)


def copy_lora(group, lora):
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)


@pytest.mark.parametrize("side_stream", [False, True])
def test_unet_context_gradient_tiny(side_stream):
    """d(ehs) in fp32 = the sum over every attn2 of its k/v dgrad (merged LoRA included), inline and hoisted k/v paths."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    _, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(group, lora)
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    G = torch.randn(lat.shape, generator=torch.Generator().manual_seed(3))
    e = ehs.to(DEV).requires_grad_(True)
    ops.set_side_stream(side_stream)
    try:
        pred = unet(lat.to(DEV), t.to(DEV), e).sample
        (pred * G.to(DEV)).sum().backward()
    finally:
        ops.join_side()
        ops.set_side_stream(False)
    assert e.grad is not None and e.grad.dtype == torch.float32
    er = ehs.clone().requires_grad_(True)
    pr = U.unet_forward(sd, lat, t, er, lora=lora, spec=spec)
    (pr * G).sum().backward()
    err = rel(e.grad, er.grad)
    print(f"[ctx grad side_stream={side_stream}] rel={err:.3e}")
    assert err <= 5e-2
    # no gradient wanted: the text embedding takes the old path (one cast, no fan-out and no summing kernel)
    before = _lib.launch_count
    with torch.no_grad():
        unet(lat.to(DEV), t.to(DEV), ehs.to(DEV))
    n_plain = _lib.launch_count - before
    before = _lib.launch_count
    with torch.no_grad():
        unet(lat.to(DEV), t.to(DEV), e)
    assert _lib.launch_count - before == n_plain


def build_joint(optimizer="adamw", clip_skip=1, max_norm=1.0, use_graph=False):
    spec, tspec = U.TINY, R.TINY_TE
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(ugroup, lora)
    tsd = R.init_params(tspec, seed=5)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=1e-5)
    tlora = R.init_lora(tspec, rank=4)
    copy_lora(tgroup, tlora)
    opts = {"n_repeats": 1, "clip_skip": clip_skip, "clip_final_norm": True}
    step = LoraTrainStep(unet, ugroups + tgroups, lr=1e-4, max_grad_norm=max_norm, use_cuda_graph=use_graph, optimizer=optimizer,
                         text_encoder=te, text_encoder_opts=opts)
    ref = R.joint_reference_loop(sd, lora, spec, tsd, tlora, tspec, opts, lr=1e-4, te_lr=1e-5, max_grad_norm=max_norm)
    return step, ref, ugroup, tgroup, lora, tlora


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("max_norm", [1.0, 1e-3])
def test_joint_te_unet_steps_match_reference_loop(use_graph, max_norm):
    """Three AdamW steps of the TINY UNet + a two-layer text encoder, both adapter sets, clip_skip 1 (the last layer's adapters get a
    zero gradient and only decay), with and without an active joint clip (max_norm 1e-3 clips every step)."""
    step, ref, ugroup, tgroup, lora, tlora = build_joint(max_norm=max_norm, use_graph=use_graph)
    spec = U.TINY
    before_u = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in ugroup.plugin_dict.items()}
    before_t = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in tgroup.plugin_dict.items()}
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, spec, seed=100 + i)
        ids = R.synthetic_ids(2, 1, seed=200 + i)
        loss = float(step.step(lat, noise, t, ids).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids)
        print(f"[joint step {i}] loss {loss:.6f} ref {loss_ref:.6f}")
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref)
    for name, group, refl, before in (("unet", ugroup, lora, before_u), ("te", tgroup, tlora, before_t)):
        got = torch.cat([torch.cat([(b.layer.W_down - before[k][0]).flatten(), (b.layer.W_up - before[k][1]).flatten()]).cpu()
                         for k, b in group.plugin_dict.items()]).double()
        want = torch.cat([torch.cat([(refl[k][0].W_down.detach() - before[k][0].cpu()).flatten(),
                                     (refl[k][0].W_up.detach() - before[k][1].cpu()).flatten()]) for k in group.plugin_dict]).double()
        cos = float(got @ want / (got.norm() * want.norm()))
        ratio = float(got.norm() / want.norm())
        print(f"[joint {name} max_norm={max_norm} graph={use_graph}] update cos {cos:.4f} norm ratio {ratio:.4f}")
        assert cos >= 0.9 and 0.9 < ratio < 1.1
    # the skipped layer's adapters (layer 1 of 2 with clip_skip 1): zero gradient, so AdamW only decays them, as in the reference
    for k, b in tgroup.plugin_dict.items():
        if ".layers.1." in k:
            for got, ref_p, b0 in ((b.layer.W_down, tlora[k][0].W_down, before_t[k][0]), (b.layer.W_up, tlora[k][0].W_up, before_t[k][1])):
                assert not torch.equal(got, b0), f"{k}: not decayed"
                assert rel(got, ref_p) <= 1e-5, k


def test_joint_te_unet_adafactor_runs_and_moves_both_sets():
    step, _, ugroup, tgroup, _, _ = build_joint(optimizer="adafactor", clip_skip=0)
    before = [b.layer.W_up.detach().clone() for g in (ugroup, tgroup) for b in g.plugin_dict.values()]
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, U.TINY, seed=100 + i)
        loss = float(step.step(lat, noise, t, R.synthetic_ids(2, 1, seed=200 + i)).cpu())
        assert loss == loss
    after = [b.layer.W_up.detach() for g in (ugroup, tgroup) for b in g.plugin_dict.values()]
    assert all(not torch.equal(a, b) for a, b in zip(after, before))


def test_refuses_uncovered_combinations():
    spec = U.TINY
    unet = tiny_unet(U.init_params(spec))
    groups, _ = make_hcpdiff(unet, None, [{"rank": 4, "layers": [r"re:.*\.attn.?$"]}])
    te = CLIPTextModel(**R.TINY_TE.kwargs()).to(DEV).requires_grad_(False)
    tgroups, _ = make_hcpdiff(te, None, [{"rank": 4, "layers": [r"re:.*self_attn$"]}])
    with pytest.raises(NotImplementedError, match="cfg_scale"):
        LoraTrainStep(unet, groups + tgroups, cfg_scale="0.5-1.0", text_encoder=te)
    with pytest.raises(ValueError, match="not in `params`"):
        LoraTrainStep(unet, groups, text_encoder=te)


TE_CFG = """
exp_dir: {exp}
seed: 3
model:
  unet:
    _target_: hcp_diffusion_b200.models.UNet2DConditionModel
    sample_size: 16
    block_out_channels: [64, 128, 128, 128]
    attention_head_dim: 2
    cross_attention_dim: 64
  text_encoder:
    _target_: hcp_diffusion_b200.models.CLIPTextModel
    hidden_size: 64
    intermediate_size: 256
    num_hidden_layers: 2
    num_attention_heads: 1
  clip_skip: 1
  tokenizer_repeats: 2
  ema: {{decay_max: 0.99}}
lora_unet:
  - {{lr: 1e-4, rank: 4, layers: ['re:.*\\\\.attn.?$']}}
lora_text_encoder:
  - {{lr: 1e-5, rank: 4, layers: ['re:.*self_attn$', 're:.*mlp$']}}
tokenizer_pt:
  train: null
train:
  train_steps: 2
  save_step: 2
  log_step: 1
data:
  batch_size: 2
  num_samples: 8
"""


def test_train_ac_text_encoder_entrypoint_saves_and_resumes(tmp_path):
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    cfg_path = os.path.join(tmp_path, "te.yaml")
    with open(cfg_path, "w") as f:
        f.write(TE_CFG.format(exp=os.path.join(tmp_path, "exp")))
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", cfg_path], cwd=ROOT, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 2/2" in r.stdout
    ck = os.path.join(tmp_path, "exp", "ckpts", "text_encoder-2.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert set(sd) == {"lora", "lora_ema"}
    assert "text_model.encoder.layers.0.self_attn.q_proj.___.layer.W_down" in sd["lora"]
    assert len([k for k in sd["lora"] if k.endswith("W_up")]) == 12
    assert os.path.exists(os.path.join(tmp_path, "exp", "ckpts", "unet-2.safetensors"))
    conf = load_config_with_cli(cfg_path, [f"train.resume.ckpt_path.TE=[{ck}]", "train.resume.start_step=2", "train.train_steps=3"])
    tr = Trainer(conf)
    live = tr.te_lora.state_dict()
    for k, v in sd["lora"].items():
        torch.testing.assert_close(live[k].cpu(), v, msg=k)
    assert tr.ehs.shape == (8, 154) and tr.ehs.dtype == torch.int64
    tr.train()
