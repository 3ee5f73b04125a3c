"""GPU tests of training LoRA on SDXL's two text encoders with the UNet (`pytest -m gpu`): the exact-GELU kernels against float64,
`encode_prompt_sdxl` with adapters on both encoders against the fp32 restatement tests/sdxl_te_ref.py (pinned to transformers + the
reference's SDXLTextEncoder / TEEXHook by tests/golden/ref_sdxl_te.pt), the UNet's gradients of text_embeds and of the context, the
joint step against the reference loop (tests/sdxl_te_ref.joint_reference_loop), bit-identical repeats and the entrypoint.

Bounds: about 2-3x the worst value measured on one H100 80GB HBM3 (700 W power limit) over the cases below.

                                                                          measured worst     bound
  GELU forward / backward, relative L2 vs fp64 on the bf16 inputs         1.51e-3            4e-3
  encode_prompt_sdxl (SMALL_XL and full size): ehs, text_embeds rel L2    1.30e-2            3e-2
  adapter gradients of both encoders, global rel L2                       1.37e-2            3.5e-2
  TINY_XL UNet with LoRA: noise_pred rel L2 vs the fp32 oracle            1.51e-2            4e-2
  TINY_XL UNet: d(text_embeds), d(ehs) rel L2 vs the fp32 oracle          5.55e-2            1.2e-1
    (d(text_embeds) is the sum over every resnet's time_emb_proj of bf16-operand products, back through add_embedding)
  joint step (as tests/test_gpu_te_step.py): loss within 2e-2 relative (measured 5.7e-4), update direction cosine >= 0.9 (measured
  >= 0.9957) and norm ratio in (0.9, 1.1) (measured 0.9994-1.0014), per model: UNet, clip_B, clip_bigG
"""
import math
import os
import subprocess
import sys

import pytest
import torch

import sdxl_te_ref as X

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib, ops  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import SDXLTextEncoder, UNet2DConditionModel, encode_prompt_sdxl  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TE_ITEM = {"lr": 1e-5, "rank": 4, "alpha": 1.0, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}

BOUND_GELU = 4e-3
BOUND_ENC = 3e-2
BOUND_GRAD = 3.5e-2
BOUND_UNET_PRED = 4e-2
BOUND_UNET_GRAD = 1.2e-1


def rel(got, ref):
    got, ref = got.detach().double().flatten().cpu(), ref.detach().double().flatten().cpu()
    return float((got - ref).norm() / (ref.norm() + 1e-30))


def copy_lora(group, lora):
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)


# ----------------------------------------------------------------------------------------------------------------------
# exact GELU
# ----------------------------------------------------------------------------------------------------------------------
def test_gelu_matches_fp64():
    g = torch.Generator().manual_seed(17)
    x = (torch.randn(308, 5120, generator=g) * 3.0)
    x[0, :16] = torch.tensor([0.0, -0.0, 5.0, -5.0, 5.5, -5.5, 8.0, -8.0, 12.0, -12.0, 40.0, -40.0, 1e-3, -1e-3, 0.5, -0.5])
    x = x.to(DEV, torch.bfloat16).requires_grad_(True)
    dy = torch.randn(308, 5120, generator=g).to(DEV, torch.bfloat16)
    y = ops.GeluFn.apply(x)
    y.backward(dy)
    xr = x.detach().to(F64).requires_grad_(True)
    yr = torch.nn.functional.gelu(xr)
    yr.backward(dy.to(F64))
    for nm, got, ref in (("y", y, yr), ("dx", x.grad, xr.grad)):
        err = rel(got, ref)
        print(f"[gelu {nm}] rel={err:.3e}")
        assert err <= BOUND_GELU
    # the tails and the signed zeros, element by element
    xs, ys, ds = x.detach()[0, :16].to(F64), y.detach()[0, :16].to(F64), x.grad[0, :16].to(F64)
    d0 = dy[0, :16].to(F64)
    assert ys[0] == 0 and ys[1] == 0 and ds[0] == 0.5 * d0[0] and ds[1] == 0.5 * d0[1]
    big = xs.abs() > 5
    assert torch.equal(ys[big & (xs > 0)], xs[big & (xs > 0)])                 # x Phi(x) rounds to x in bf16
    assert float(ys[big & (xs < 0)].abs().max()) < 1e-5                         # the negative tail vanishes
    assert torch.allclose(ds[big & (xs > 0)], d0[big & (xs > 0)], rtol=8e-3)
    assert float(ds[big & (xs < 0)].abs().max()) < 1e-5


# ----------------------------------------------------------------------------------------------------------------------
# encode_prompt_sdxl with adapters on both encoders
# ----------------------------------------------------------------------------------------------------------------------
def build_pair(pair, seed=0, rank=4):
    sd = X.init_params(pair, seed)
    te = SDXLTextEncoder(**pair.kwargs())
    te.load_state_dict(sd)
    te = te.requires_grad_(False).to(DEV)
    _, group = make_hcpdiff(te, None, [dict(TE_ITEM, rank=rank)])
    lora = X.init_lora(pair, rank)
    copy_lora(group, lora)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    lora_dev = {k: [U.LoraEntry(e.W_down.to(DEV).requires_grad_(True), e.W_up.to(DEV).requires_grad_(True), e.alpha, None) for e in v]
                for k, v in lora.items()}
    return te, group, sd_dev, lora_dev


@pytest.mark.parametrize("pair_name,batch,clip_skip,final_norm", [
    ("SMALL_XL", 2, 0, True), ("SMALL_XL", 2, 1, False), ("SMALL_XL", 20, 1, False), ("FULL", 2, 1, False)])
def test_encode_prompt_sdxl_and_adapter_grads(pair_name, batch, clip_skip, final_norm):
    """Batch 20 runs the projection GEMM above the 16 rows of the skinny linear; FULL is CLIP-L + OpenCLIP-bigG at full size."""
    pair = getattr(X, pair_name)
    te, group, sd, lora = build_pair(pair)
    ids = X.synthetic_ids(batch, seed=21).to(DEV)
    with torch.no_grad():
        ehs_ng, emb_ng = encode_prompt_sdxl(te, ids, clip_skip, final_norm)
    ehs, emb = encode_prompt_sdxl(te, ids, clip_skip, final_norm)
    ehs_ref, emb_ref = X.encode_prompt_sdxl(sd, ids, pair, clip_skip, final_norm, lora)
    C_ = pair.clip_B.hidden_size + pair.clip_bigG.hidden_size
    assert ehs.shape == ehs_ref.shape == (batch, 77, C_) and ehs.dtype == torch.bfloat16
    assert emb.shape == emb_ref.shape == (batch, pair.projection_dim) and emb.dtype == torch.float32
    errs = {"ehs": rel(ehs.float(), ehs_ref), "text_embeds": rel(emb, emb_ref), "ehs no_grad": rel(ehs_ng.float(), ehs_ref),
            "text_embeds no_grad": rel(emb_ng, emb_ref)}
    print(f"[{pair_name} B{batch} skip{clip_skip} norm{int(final_norm)}] " + ", ".join(f"{k} {v:.3e}" for k, v in errs.items()))
    assert max(errs.values()) <= BOUND_ENC
    g = torch.Generator().manual_seed(5)
    G1 = torch.randn(ehs.shape, generator=g).to(DEV)
    G2 = torch.randn(emb.shape, generator=g).to(DEV)
    ((ehs.float() * G1).sum() + (emb * G2).sum()).backward()
    ((ehs_ref * G1).sum() + (emb_ref * G2).sum()).backward()
    num = den = 0.0
    n_b = pair.clip_B.num_hidden_layers - clip_skip
    for layer, entries in lora.items():
        blk = group[layer].layer
        idx = int(layer.split(".")[4])
        for got, ref_p in ((blk.W_down.grad, entries[0].W_down), (blk.W_up.grad, entries[0].W_up)):
            if layer.startswith("clip_B.") and idx >= n_b:       # clip_B's layers after the taken hidden state: no gradient
                assert got is None or not got.any(), layer
                continue
            assert got is not None, layer                        # every bigG layer, the last through text_embeds
            num += float((got.double() - ref_p.grad.double()).pow(2).sum())
            den += float(ref_p.grad.double().pow(2).sum())
    ge = math.sqrt(num / den)
    print(f"[{pair_name} B{batch} skip{clip_skip}] adapter grads global rel={ge:.3e}")
    assert ge <= BOUND_GRAD


# ----------------------------------------------------------------------------------------------------------------------
# the UNet's gradient of text_embeds
# ----------------------------------------------------------------------------------------------------------------------
def tiny_xl_unet(sd):
    spec = U.TINY_XL
    down = tuple("CrossAttnDownBlock2D" if a else "DownBlock2D" for a in spec.down_has_attn)
    up = tuple("CrossAttnUpBlock2D" if a else "UpBlock2D" for a in spec.up_has_attn)
    u = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
                             cross_attention_dim=spec.cross_attention_dim, down_block_types=down, up_block_types=up,
                             transformer_layers_per_block=spec.transformer_depth, use_linear_projection=True,
                             addition_embed_type="text_time", addition_time_embed_dim=spec.addition_time_embed_dim,
                             projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)
    u.load_state_dict(sd)
    return u.to(DEV).requires_grad_(False)


def test_tiny_xl_text_embeds_and_context_gradients():
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet = tiny_xl_unet(sd)
    _, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(group, lora)
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    added = U.synthetic_added_cond(2, spec)
    G = torch.randn(lat.shape, generator=torch.Generator().manual_seed(3))
    e = ehs.to(DEV).requires_grad_(True)
    te_ = added["text_embeds"].to(DEV).requires_grad_(True)
    pred = unet(lat.to(DEV), t.to(DEV), e, added_cond_kwargs={"text_embeds": te_, "time_ids": added["time_ids"].to(DEV)}).sample
    (pred * G.to(DEV)).sum().backward()
    assert te_.grad is not None and te_.grad.dtype == torch.float32
    assert all(p.grad is None for n, p in unet.named_parameters() if n.startswith("add_embedding."))     # stays frozen
    er, tr = ehs.clone().requires_grad_(True), added["text_embeds"].clone().requires_grad_(True)
    pr = U.unet_forward(sd, lat, t, er, lora=lora, spec=spec, added_cond_kwargs={"text_embeds": tr, "time_ids": added["time_ids"]})
    (pr * G).sum().backward()
    errs = {"pred": rel(pred, pr), "d(text_embeds)": rel(te_.grad, tr.grad), "d(ehs)": rel(e.grad, er.grad)}
    print("[TINY_XL] " + ", ".join(f"{k} {v:.3e}" for k, v in errs.items()))
    assert errs["pred"] <= BOUND_UNET_PRED and max(errs["d(text_embeds)"], errs["d(ehs)"]) <= BOUND_UNET_GRAD
    # without a text-embedding gradient the fused add_embedding path runs: the same launches as a plain no-grad forward
    a_dev = {k: v.to(DEV) for k, v in added.items()}
    before = _lib.launch_count
    with torch.no_grad():
        unet(lat.to(DEV), t.to(DEV), ehs.to(DEV), added_cond_kwargs=a_dev)
    n_plain = _lib.launch_count - before
    before = _lib.launch_count
    with torch.no_grad():
        unet(lat.to(DEV), t.to(DEV), ehs.to(DEV), added_cond_kwargs={"text_embeds": te_, "time_ids": a_dev["time_ids"]})
    assert _lib.launch_count - before == n_plain


# ----------------------------------------------------------------------------------------------------------------------
# joint steps
# ----------------------------------------------------------------------------------------------------------------------
AF_KW = {"lr": 1e-3, "relative_step": False, "beta1": 0.9, "weight_decay": 1e-2}


def build_joint(optimizer="adamw", clip_skip=1, final_norm=False, use_graph=True, max_norm=1.0):
    spec, pair = U.TINY_XL, X.TINY_XL_TE
    sd = U.init_params(spec)
    unet = tiny_xl_unet(sd)
    ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(ugroup, lora)
    tsd = X.init_params(pair, seed=5)
    te = SDXLTextEncoder(**pair.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [dict(TE_ITEM)], default_lr=1e-5)
    tlora = X.init_lora(pair, rank=4)
    copy_lora(tgroup, tlora)
    opts = {"clip_skip": clip_skip, "clip_final_norm": final_norm}
    af = AF_KW if optimizer == "adafactor" else None
    step = LoraTrainStep(unet, ugroups + tgroups, lr=1e-4, max_grad_norm=max_norm, use_cuda_graph=use_graph, optimizer=optimizer,
                         optimizer_kwargs=af, text_encoder=te, text_encoder_opts=opts)
    ref = X.joint_reference_loop(sd, lora, spec, tsd, tlora, pair, clip_skip, final_norm, lr=1e-4, te_lr=1e-5, optimizer_kwargs=af,
                                 max_grad_norm=max_norm)
    return step, ref, ugroup, tgroup, lora, tlora


def batch(i):
    lat, noise, t, _ = U.synthetic_batch(2, U.TINY_XL, seed=100 + i)
    return lat, noise, t, X.synthetic_ids(2, seed=200 + i), U.synthetic_added_cond(2, U.TINY_XL, seed=300 + i)["time_ids"]


@pytest.mark.parametrize("optimizer,clip_skip,final_norm,use_graph", [
    ("adamw", 1, False, True), ("adamw", 0, True, False), ("adafactor", 1, False, True), ("adafactor", 0, True, True)])
def test_joint_sdxl_te_unet_steps_match_reference_loop(optimizer, clip_skip, final_norm, use_graph):
    step, ref, ugroup, tgroup, lora, tlora = build_joint(optimizer, clip_skip, final_norm, use_graph)
    before_u = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in ugroup.plugin_dict.items()}
    before_t = {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in tgroup.plugin_dict.items()}
    for i in range(3):
        lat, noise, t, ids, time_ids = batch(i)
        loss = float(step.step(lat, noise, t, ids, {"time_ids": time_ids}).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids, time_ids)
        print(f"[joint {optimizer} skip{clip_skip} step {i}] loss {loss:.6f} ref {loss_ref:.6f}")
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref)
    for name, group, refl, before, sel in (("unet", ugroup, lora, before_u, None), ("clip_B", tgroup, tlora, before_t, "clip_B."),
                                           ("clip_bigG", tgroup, tlora, before_t, "clip_bigG.")):
        keys = [k for k in group.plugin_dict if sel is None or k.startswith(sel)]
        got = torch.cat([torch.cat([(group.plugin_dict[k].layer.W_down - before[k][0]).flatten(),
                                    (group.plugin_dict[k].layer.W_up - before[k][1]).flatten()]).cpu() for k in keys]).double()
        want = torch.cat([torch.cat([(refl[k][0].W_down.detach() - before[k][0].cpu()).flatten(),
                                     (refl[k][0].W_up.detach() - before[k][1].cpu()).flatten()]) for k in keys]).double()
        cos = float(got @ want / (got.norm() * want.norm()))
        ratio = float(got.norm() / want.norm())
        print(f"[joint {optimizer} skip{clip_skip} {name}] update cos {cos:.4f} norm ratio {ratio:.4f}")
        assert cos >= 0.9 and 0.9 < ratio < 1.1
    # bigG's last layer with clip_skip 1: trained through text_embeds alone, and it moves like the reference's
    last = f"clip_bigG.text_model.encoder.layers.{X.TINY_XL_TE.clip_bigG.num_hidden_layers - 1}.mlp.fc2"
    moved = tgroup.plugin_dict[last].layer.W_up - before_t[last][1]
    want = tlora[last][0].W_up.detach() - before_t[last][1].cpu()
    assert float(moved.norm()) > 0 and rel(moved, want) < 0.3


def test_gelu_and_encoder_forward_are_bit_identical():
    """The GELU kernels and the pair's forward repeat bit for bit (the step's gradient reductions, loss and clip norm use fp32
    atomics, DESIGN.md section 7, so the step as a whole is not asserted)."""
    x = (torch.randn(77 * 20, 512, generator=torch.Generator().manual_seed(3)) * 4).to(DEV, torch.bfloat16)
    dy = torch.randn(77 * 20, 512, generator=torch.Generator().manual_seed(4)).to(DEV, torch.bfloat16)
    te, _, _, _ = build_pair(X.SMALL_XL)
    ids = X.synthetic_ids(20, seed=9).to(DEV)
    runs = []
    for _ in range(3):
        xg = x.clone().requires_grad_(True)
        y = ops.GeluFn.apply(xg)
        y.backward(dy)
        ehs, emb = encode_prompt_sdxl(te, ids, 1, False)
        runs.append([t.detach().clone() for t in (y, xg.grad, ehs, emb)])
    for again in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], again))


# ----------------------------------------------------------------------------------------------------------------------
# entrypoint
# ----------------------------------------------------------------------------------------------------------------------
def test_train_ac_sdxl_te_yaml_on_tiny_xl_saves_and_resumes(tmp_path):
    """cfgs/train/lora_sdxl_te_synthetic.yaml with the UNet and the text encoders shrunk to TINY_XL / TINY_XL_TE."""
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    spec, pair = U.TINY_XL, X.TINY_XL_TE
    cfg = os.path.join(ROOT, "cfgs/train/lora_sdxl_te_synthetic.yaml")
    exp = os.path.join(tmp_path, "exp")
    b, g = pair.clip_B, pair.clip_bigG
    over = [f"exp_dir={exp}", "train.train_steps=2", "train.save_step=2", "train.log_step=1", "data.batch_size=2", "data.num_samples=8",
            f"model.unet.sample_size={spec.sample_size}", "model.unet.block_out_channels=[64,128,128]",
            "model.unet.attention_head_dim=[1,2,2]", f"model.unet.cross_attention_dim={spec.cross_attention_dim}",
            "model.unet.transformer_layers_per_block=[1,2,3]", f"model.unet.addition_time_embed_dim={spec.addition_time_embed_dim}",
            f"model.unet.projection_class_embeddings_input_dim={spec.projection_class_embeddings_input_dim}",
            "model.text_encoder._target_=hcp_diffusion_b200.models.SDXLTextEncoder",
            *(f"model.text_encoder.{name}={{" + ", ".join(f"{k}: {v}" for k, v in kw.items() if k != "layer_norm_eps") + "}"
              for name, kw in pair.kwargs().items()),
            "model.ema={decay_max: 0.99}"]
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", cfg, *over], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 2/2" in r.stdout
    ck = os.path.join(exp, "ckpts", "text_encoder-2.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert set(sd) == {"lora", "lora_ema"}
    assert "clip_B.text_model.encoder.layers.0.self_attn.q_proj.___.layer.W_down" in sd["lora"]
    assert "clip_bigG.text_model.encoder.layers.2.mlp.fc2.___.layer.W_up" in sd["lora"]
    n_linears = 6 * (b.num_hidden_layers + g.num_hidden_layers)
    assert len([k for k in sd["lora"] if k.endswith("W_up")]) == n_linears
    assert os.path.exists(os.path.join(exp, "ckpts", "unet-2.safetensors"))
    conf = load_config_with_cli(cfg, over + [f"train.resume.ckpt_path.TE=[{ck}]", "train.resume.start_step=2", "train.train_steps=3"])
    tr = Trainer(conf)
    live = tr.te_lora.state_dict()
    for k, v in sd["lora"].items():
        torch.testing.assert_close(live[k].cpu(), v, msg=k)
    assert tr.ehs.shape == (8, 154) and tr.ehs.dtype == torch.int64
    ids_b, ids_g = tr.ehs[:, :77], tr.ehs[:, 77:]             # the same words; bigG's chunk has one EOS, then id 0 padding
    eos = (ids_b == X.EOS).int().argmax(1)
    assert bool(((ids_g == X.EOS).sum(1) == 1).all()) and torch.equal(ids_g.argmax(1), eos) and torch.equal(ids_b.argmax(1), eos)
    assert all(bool((ids_g[r, eos[r] + 1:] == 0).all()) and torch.equal(ids_g[r, :eos[r]], ids_b[r, :eos[r]]) for r in range(8))
    assert tr.text_embeds is None
    tr.train()
