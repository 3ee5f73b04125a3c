"""Adafactor on the GPU: the kernels against the fp64 restatement on every shape class, determinism and stray writes; SDXL full
fine-tuning of TINY_XL (every gradient, including the time and additional embeddings, and add_embedding trained with the time path
frozen); optimizer steps of the engine against the reference loop with Adafactor; the training entrypoint on a TINY_XL copy of
cfgs/train/ft_sdxl_synthetic.yaml; SDXL-base at 1024 px.

Kernel bounds: per tensor, the update p_new - p_old beyond one fp32 ulp of the stored parameter (an update of 1e-4 on a parameter
of magnitude 1 is only resolved to about 6e-4 by the fp32 store itself), and each state, as rel-L2 against fp64 over 8 steps.
Bounds are about 3x the worst case measured on an H100 80GB HBM3 (700 W): update 3.6e-7, state 1.5e-6 (exp_avg of the 1-element
tensor)."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import adafactor as A  # noqa: E402
from hcp_diffusion_b200._lib import call, ptr, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

import adafactor_ref as R  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SHAPES = R.GOLDEN_SHAPES + [(1280, 5120), (10240, 1280), (320, 4, 3, 3), (1280, 640, 1, 1)]
GROUP_OPTS = [{}, {"lr": 1e-3, "relative_step": False, "scale_parameter": False, "beta1": 0.9, "weight_decay": 1e-3}]
DELTA_BOUND, STATE_BOUND = 1e-6, 5e-6


def rel_l2(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


class FlatAdafactor:
    """The kernels on a hand-built flat buffer: tensor i in group i % 2, the padding filled with a sentinel."""

    def __init__(self, shapes, seed=0):
        self.shapes = shapes
        self.offs, n = [], 0
        for s in shapes:
            self.offs.append(n)
            n += (math.prod(s) + 3) // 4 * 4
        self.groups = [i % 2 for i in range(len(shapes))]
        self.lay = A.Layout(shapes, self.offs, self.groups)
        g = torch.Generator().manual_seed(seed)
        self.p = torch.full((n,), 7.25)
        for s, o in zip(shapes, self.offs):
            self.p[o:o + math.prod(s)] = torch.randn(math.prod(s), generator=g)
        self.p = self.p.to(DEV)
        self.state = torch.zeros(self.lay.state_numel, device=DEV)
        self.m = torch.zeros(n, device=DEV)
        self.work = torch.zeros(self.lay.work_numel, device=DEV)
        opts = [A.check_options(o) for o in GROUP_OPTS]
        self.hyper = torch.tensor([A.hyper_row(o, o["lr"], o["weight_decay"]) for o in opts], device=DEV)
        self.steps = torch.zeros(2, dtype=torch.int32, device=DEV)
        to_dev = lambda a: torch.from_numpy(a.view(np.uint8).copy()).to(DEV)  # noqa: E731
        self.tt, self.it, self.fi = to_dev(self.lay.tensors), to_dev(self.lay.items), to_dev(self.lay.factor_items)

    def step(self, grad, gscale, max_norm):
        gsq = torch.zeros(1, device=DEV)
        call("hcp_sumsq", grad.data_ptr(), grad.numel(), gsq.data_ptr(), stream_ptr())
        call("hcp_adafactor_flat", self.p.data_ptr(), grad.data_ptr(), self.state.data_ptr(), self.m.data_ptr(), self.work.data_ptr(),
             self.tt.data_ptr(), self.it.data_ptr(), self.lay.items.size, ptr(self.fi), self.lay.factor_items.size, self.hyper.data_ptr(),
             self.steps.data_ptr(), 2, gscale, gsq.data_ptr(), max_norm, stream_ptr())

    def view(self, buf, i):
        o = self.offs[i]
        return buf[o:o + math.prod(self.shapes[i])].view(self.shapes[i])

    def states(self, i):
        t = self.lay.tensors[i]
        if t["factored"]:
            P, Rr, C = (int(x) for x in (t["P"], t["R"], t["C"]))
            s = self.shapes[i]
            return {"exp_avg_sq_row": self.state[t["row"]:t["row"] + P * Rr].view(s[:-1]),
                    "exp_avg_sq_col": self.state[t["col"]:t["col"] + P * C].view(s[:-2] + s[-1:])}
        return {"exp_avg_sq": self.state[t["row"]:t["row"] + int(t["numel"])].view(self.shapes[i])}


def grads_for(fa, step, seed=100):
    g = torch.Generator().manual_seed(seed + step)
    grad = torch.zeros(fa.p.numel())
    for s, o in zip(fa.shapes, fa.offs):
        grad[o:o + math.prod(s)] = torch.randn(math.prod(s), generator=g) * (1.0 if step < 5 else 30.0)
    return grad.to(DEV)


def test_kernels_match_fp64_oracle_every_shape():
    fa = FlatAdafactor(KERNEL_SHAPES)
    gscale, max_norm = 0.5, 1.0
    pad_mask = torch.ones(fa.p.numel(), dtype=torch.bool)
    for s, o in zip(fa.shapes, fa.offs):
        pad_mask[o:o + math.prod(s)] = False
    ref_p = [fa.view(fa.p, i).double().cpu().clone() for i in range(len(fa.shapes))]
    ref_state = [{} for _ in fa.shapes]
    worst = {}
    for k in range(8):
        grad = grads_for(fa, k)
        grad_before = grad.clone()
        p_before = [fa.view(fa.p, i).double().cpu().clone() for i in range(len(fa.shapes))]
        fa.step(grad, gscale, max_norm)
        torch.cuda.synchronize()
        assert torch.equal(grad, grad_before)                          # the gradient is read only
        norm = float(grad.double().norm()) * gscale
        clip = min(1.0, max_norm / (norm + 1e-6))
        assert clip < 1.0                                              # the global clip is active
        for i, s in enumerate(fa.shapes):
            g = fa.view(grad, i).double().cpu() * gscale * clip
            opts = A.check_options(GROUP_OPTS[fa.groups[i]])
            opts = {k2: v for k2, v in opts.items() if k2 != "lr"}
            pre = ref_p[i].clone()
            R.adafactor_step(ref_p[i], g, ref_state[i], lr=GROUP_OPTS[fa.groups[i]].get("lr"), **opts)
            d_ref = ref_p[i] - pre
            p_new = fa.view(fa.p, i).cpu()
            d_got = p_new.double() - p_before[i]
            ulp = torch.from_numpy(np.spacing(np.abs(p_new.numpy()))).double()
            e = float((d_got - d_ref).abs().sub(ulp).clamp(min=0).norm() / (d_ref.norm() + 1e-30))
            worst[("delta", s)] = max(worst.get(("delta", s), 0.0), e)
            got_states = fa.states(i)
            if fa.groups[i] == 1:
                got_states["exp_avg"] = fa.view(fa.m, i)
            for name, v in got_states.items():
                es = rel_l2(v, ref_state[i][name])
                worst[(name, s)] = max(worst.get((name, s), 0.0), es)
            # continue from the kernel's parameters so that the two trajectories do not drift apart
            ref_p[i] = fa.view(fa.p, i).double().cpu().clone()
    print("worst per tensor:", sorted(worst.items(), key=lambda kv: -kv[1]))
    assert bool(torch.all(fa.p.cpu()[pad_mask] == 7.25))               # the padding between tensors is never written
    assert int(fa.steps.cpu()[0]) == 8
    for (name, s), e in worst.items():
        assert e < (DELTA_BOUND if name == "delta" else STATE_BOUND), (name, s, e)


def test_kernels_are_deterministic():
    """Bit-identical repeats.  Without the global clip: hcp_sumsq (the clip's norm, shared with AdamW) sums with atomics, so its
    last bits -- and through the clip factor every update -- may differ between runs; the Adafactor passes themselves have
    fixed-order reductions only."""
    runs = []
    for _ in range(2):
        fa = FlatAdafactor(KERNEL_SHAPES, seed=3)
        for k in range(3):
            fa.step(grads_for(fa, k, seed=7), 1.0, 0.0)
        runs.append((fa.p.cpu(), fa.state.cpu(), fa.m.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def unet_for_spec(spec):
    down = tuple("CrossAttnDownBlock2D" if a else "DownBlock2D" for a in spec.down_has_attn)
    up = tuple("CrossAttnUpBlock2D" if a else "UpBlock2D" for a in spec.up_has_attn)
    return UNet2DConditionModel(
        sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
        cross_attention_dim=spec.cross_attention_dim, down_block_types=down, up_block_types=up,
        transformer_layers_per_block=spec.transformer_depth, use_linear_projection=spec.use_linear_projection,
        addition_embed_type="text_time" if spec.addition_time_embed_dim else None, addition_time_embed_dim=spec.addition_time_embed_dim,
        projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)


def full_ft_xl(sd):
    unet = unet_for_spec(U.TINY_XL)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-5, "layers": [""]}], None)
    assert lora.empty() and len(groups) == 1
    return unet, groups


def test_tiny_xl_full_finetune_every_gradient_matches_oracle():
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet, groups = full_ft_xl(sd)
    assert all(p.requires_grad for p in unet.parameters())
    step = LoraTrainStep(unet, groups, use_cuda_graph=False, optimizer="adafactor")
    lat, noise, t, ehs = U.synthetic_batch(4, spec)
    added = U.synthetic_added_cond(4, spec)
    step._forward_backward(lat.to(DEV), noise.to(DEV), t.to(DEV), ehs.to(DEV), {k: v.to(DEV) for k, v in added.items()})
    torch.cuda.synchronize()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    x_t = U.add_noise(lat, noise, t, U.ddpm_alphas_cumprod())
    pred = U.unet_forward(ref_sd, x_t, t, ehs, spec=spec, added_cond_kwargs=added)
    F.mse_loss(pred, noise, reduction="none").mean().backward()
    num = den = 0.0
    emb = {}
    for name, p in unet.named_parameters():
        ref = ref_sd[name].grad
        assert ref is not None and p.grad is not None, name
        num += float((p.grad.cpu().double() - ref.double()).pow(2).sum())
        den += float(ref.double().pow(2).sum())
        if name.startswith(("time_embedding.", "add_embedding.")):
            emb[name] = rel_l2(p.grad, ref)
    print("embedding gradients:", emb, "global", math.sqrt(num / den))
    assert len(emb) == 8 and all(e < 5e-2 for e in emb.values())
    assert math.sqrt(num / den) < 5e-2


def test_tiny_xl_add_embedding_trained_with_frozen_time_path():
    """Only add_embedding (and the attention layers) trained: the time MLP and every time_emb_proj stay frozen, and dL/demb must
    still reach the four add_embedding tensors."""
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet = unet_for_spec(spec)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-5, "layers": ["add_embedding", r"re:.*\.attn.?$"]}], None)
    trained = {n for n, p in unet.named_parameters() if p.requires_grad}
    add_names = {n for n in trained if n.startswith("add_embedding.")}
    assert len(add_names) == 4 and not any(n.startswith(("time_embedding.", "conv_in")) or "time_emb_proj" in n for n in trained)
    step = LoraTrainStep(unet, groups, use_cuda_graph=False, optimizer="adafactor")
    lat, noise, t, ehs = U.synthetic_batch(4, spec)
    added = U.synthetic_added_cond(4, spec)
    step._forward_backward(lat.to(DEV), noise.to(DEV), t.to(DEV), ehs.to(DEV), {k: v.to(DEV) for k, v in added.items()})
    torch.cuda.synchronize()
    ref_sd = {k: v.clone().requires_grad_(k in trained) for k, v in sd.items()}
    x_t = U.add_noise(lat, noise, t, U.ddpm_alphas_cumprod())
    F.mse_loss(U.unet_forward(ref_sd, x_t, t, ehs, spec=spec, added_cond_kwargs=added), noise, reduction="none").mean().backward()
    params = dict(unet.named_parameters())
    errs = {n: rel_l2(params[n].grad, ref_sd[n].grad) for n in sorted(add_names)}
    print("add_embedding gradients:", errs)
    assert all(float(params[n].grad.abs().max()) > 0 for n in add_names)
    assert all(e < 5e-2 for e in errs.values())
    num = sum(float((params[n].grad.cpu().double() - ref_sd[n].grad.double()).pow(2).sum()) for n in trained)
    den = sum(float(ref_sd[n].grad.double().pow(2).sum()) for n in trained)
    assert math.sqrt(num / den) < 5e-2


def update_check(du_p, du_r):
    cos = float((du_p.double() @ du_r.double()) / (du_p.double().norm() * du_r.double().norm()))
    ratio = float(du_p.norm() / du_r.norm())
    print("update cosine", cos, "norm ratio", ratio)
    assert cos > 0.9 and 0.9 < ratio < 1.1


AF_KW = {"lr": 1e-4, "relative_step": False, "weight_decay": 1e-3}


def test_tiny_xl_adafactor_graph_steps_match_reference_loop():
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet, groups = full_ft_xl(sd)
    names = [n for n, _ in unet.named_parameters()]
    ref_sd = {k: v.clone() for k, v in sd.items()}
    ref = R.reference_loop(ref_sd, None, spec, optimizer_kwargs=AF_KW, train_base=names)
    p0 = {n: p.detach().clone() for n, p in unet.named_parameters()}
    step = LoraTrainStep(unet, [{"params": groups[0]["params"]}], optimizer="adafactor", optimizer_kwargs=AF_KW)
    assert step.m is None and step.af_exp_avg is None
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=300 + it)
        added = U.synthetic_added_cond(4, spec, seed=50 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs, added_cond_kwargs=added)
        l_prod = float(step.step(lat, noise, t, ehs, added).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    update_check(torch.cat([(p.detach() - p0[n]).flatten().cpu() for n, p in unet.named_parameters()]),
                 torch.cat([(ref_sd[n].detach() - sd[n]).flatten() for n in names]))


def test_tiny_lora_adafactor_graph_steps_match_reference_loop():
    spec = U.TINY
    sd = U.init_params(spec)
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    _, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)
    kw = {"beta1": 0.9}                                     # relative_step (the transformers default), with a first moment
    ref = R.reference_loop(sd, lora, spec, optimizer_kwargs=kw)
    leaves = [p for layer in lora for e in lora[layer] for p in (e.W_down, e.W_up)]
    prods = [p for layer in lora for blk in [group[layer].layer] for p in (blk.W_down, blk.W_up)]
    r0, q0 = [p.detach().clone() for p in leaves], [p.detach().clone() for p in prods]
    step = LoraTrainStep(unet, prods, optimizer="adafactor", optimizer_kwargs=kw)
    assert step.af_exp_avg is not None
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=400 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref)
    update_check(torch.cat([(p.detach() - q).flatten().cpu() for p, q in zip(prods, q0)]),
                 torch.cat([(p.detach() - q).flatten() for p, q in zip(leaves, r0)]))


def test_adafactor_graph_replay_matches_eager():
    spec = U.TINY_XL
    sd = U.init_params(spec)
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    added = U.synthetic_added_cond(2, spec)
    out = []
    for use_graph in (False, True):
        unet, groups = full_ft_xl(sd)
        step = LoraTrainStep(unet, groups, use_cuda_graph=use_graph, optimizer="adafactor",
                             optimizer_kwargs={"beta1": 0.9}, ema={"decay_max": 0.999})
        losses = [float(step.step(lat, noise, t, ehs, added).cpu()) for _ in range(3)]
        out.append((losses, step.flat.data.clone(), step.af_state.clone(), int(step.af_steps[0])))
    (l0, p0, s0, n0), (l1, p1, s1, n1) = out
    assert n0 == n1 == 3
    assert np.allclose(l0, l1, rtol=1e-3, atol=0)
    # the states are EMAs of squared gradients: the run-to-run noise of the gradients (atomics in the backward) shows doubled
    assert rel_l2(p1, p0) < 1e-4 and rel_l2(s1, s0) < 2e-2


def test_train_ac_runs_tiny_xl_copy_of_ft_sdxl_yaml(tmp_path):
    import yaml
    from hcp_diffusion_b200 import train_ac
    with open(os.path.join(ROOT, "cfgs", "train", "ft_sdxl_synthetic.yaml")) as f:
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
    path = tmp_path / "ft_tiny_xl.yaml"
    path.write_text(yaml.safe_dump(cfg))
    train_ac.main(["--cfg", str(path)])
    ckpts = os.listdir(tmp_path / "exp" / "ckpts")
    assert any(c.endswith(".safetensors") for c in ckpts), ckpts


def test_sdxl_base_full_finetune_adafactor_at_1024():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_sdxl.py"), "--full-ft", "--optimizer", "adafactor",
                        "--batch", "1", "--steps", "2"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    print(line)
    assert line["optimizer_state_bytes"] == 4 * 244_330_500 and "1024x1024" in line["workload"]
    assert math.isfinite(line["loss"])
