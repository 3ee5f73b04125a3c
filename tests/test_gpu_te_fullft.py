"""GPU tests of full fine-tuning of the text encoder (`text_encoder:` items, `pytest -m gpu`): the embedding-gradient kernel
(hcp_embed_grad_bf16) bit for bit against an fp32 restatement of its documented summation order and against float64, every
parameter gradient of a trained text encoder against fp32 autograd of tests/clip_ref.py / tests/sdxl_te_ref.py, joint steps with the
UNet against the reference loop, and the entry point with cfgs/train/dreambooth_te_sd15_synthetic.yaml.

Bounds (measured on one H100 80GB HBM3 at a 700 W power limit):
  kernel: bit-identical to the fp32 restatement; against float64 |err| <= (n + 1) 2^-24 (|dst0| + sum |dH|) per element, n the rows
  of that table row (the bound of any fp32 sum of n + 1 terms); measured at most 0.50 of the bound.
  parameter gradients, relative L2 per tensor <= 5e-2 (tests/test_gpu_fullft.py's bound; bf16 activations, fp32 accumulation);
  measured at most 1.8e-2 (TINY_TE, every case), 1.6e-2 (full fine-tune + LoRA on the same layers), 1.7e-2 (TINY SDXL pair).
  joint steps, as tests/test_gpu_te_step.py: loss within 2e-2 relative, update cosine >= 0.9 and norm ratio in (0.9, 1.1) per model;
  measured cosines 0.9962-0.9998 and ratios 0.9994-1.0006 (eager and graph agree to the printed digits).
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

import clip_ref as R
import sdxl_te_ref as X

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, SDXLTextEncoder, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.models.clip import encode_prompt, encode_prompt_sdxl  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

import adafactor_ref as AF  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 32                                 # kEmbChunk of csrc/norms.cu: the piece length of the documented order


def rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---------------------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def keys_of(ids, pos_ids, V, P):
    B, L = ids.shape
    tok = np.clip(ids.reshape(-1), 0, V - 1)
    pos = np.arange(L) if pos_ids is None else pos_ids
    return tok, np.tile(np.clip(pos, 0, P - 1), B)


def restate(keys, dH, dst0):
    """The documented order in fp32: rows of one table row in row order, cut at every multiple of 32 of their position in the stable
    (key, row) order, each piece summed from 0, the pieces added in order, the total added to the table row.  Also the float64 sum
    and the per-row bound sum |dst0| + sum |dH| with the row counts."""
    order = np.argsort(keys, kind="stable")
    sk = keys[order]
    out, out64 = dst0.copy(), dst0.astype(np.float64)
    mag, cnt = np.abs(dst0).astype(np.float64), np.zeros(dst0.shape[0], np.int64)
    a = 0
    while a < len(sk):
        b = a
        while b < len(sk) and sk[b] == sk[a]:
            b += 1
        k = sk[a]
        total, lo = None, a
        while lo < b:
            hi = min(b, (lo // CHUNK + 1) * CHUNK)
            s = np.zeros(dH.shape[1], np.float32)
            for j in range(lo, hi):
                s = s + dH[order[j]]
            total = s if total is None else total + s
            lo = hi
        out[k] = out[k] + total
        rows = dH[order[a:b]].astype(np.float64)
        out64[k] += rows.sum(0)
        mag[k] += np.abs(rows).sum(0)
        cnt[k] = b - a
        a = b
    return out, out64, mag, cnt


def call_grad(ids, pos_ids, dH, dtok, dpos, V, P, ws=None):
    B, L = ids.shape
    C_ = dH.shape[-1]
    if ws is None:
        nbytes = _lib.lib().hcp_embed_grad_workspace_bytes(B, L, C_)
        ws = torch.empty(((nbytes + 15) // 16 * 4,), dtype=torch.float32, device=DEV)
    return _lib.lib().hcp_embed_grad_bf16(ids.data_ptr(), _lib.ptr(pos_ids), dH.data_ptr(), B, L, C_, _lib.ptr(dtok), V, _lib.ptr(dpos), P,
                                          ws.data_ptr(), ws.numel() * 4, stream_ptr())


def make_ids(kind, B, L, V, g):
    if kind == "equal":
        return torch.full((B, L), 7, dtype=torch.int64)
    if kind == "eos":                       # SD1.x prompts: BOS, a few words, EOS padding (EOS clamps to V - 1 on a small table)
        ids = R.synthetic_ids(B * L // 77, 1, seed=int(g.initial_seed()) % 1000).reshape(B, L)
        return ids
    if kind == "edges":                     # 0, V - 1 and ids outside the table on both sides
        choices = torch.tensor([0, V - 1, -1, -(1 << 40), V, V + 12345, 1 << 50, 3])
        return choices[torch.randint(0, len(choices), (B, L), generator=g)]
    return torch.randint(0, V, (B, L), generator=g, dtype=torch.int64)


# (name, B, L, C, V, P, ids kind, pos kind): pos kind None = absent, 'dup' = given with repeats and out-of-range entries
KERNEL_CASES = [
    ("one_row", 1, 1, 72, 50, 1, "random", None),
    ("equal_4k", 4, 1024, 72, 50, 1024, "equal", None),
    ("eos_bs16_r3", 48, 77, 768, 49408, 77, "eos", None),
    ("eos_bigG", 16, 77, 1280, 49408, 77, "eos", None),
    ("edges_pos_dup", 6, 77, 72, 300, 77, "edges", "dup"),
    ("random_small_vocab", 5, 77, 768, 40, 77, "random", None),
    ("random_pos_given", 3, 77, 1280, 1000, 100, "random", "dup"),
    ("random_3999", 3999, 1, 72, 4000, 1, "random", None),
]


def kernel_inputs(case, seed=0):
    name, B, L, C_, V, P, ids_kind, pos_kind = case
    g = torch.Generator().manual_seed(seed + 17)
    ids = make_ids(ids_kind, B, L, V, g)
    pos = None
    if pos_kind == "dup":
        pos = torch.randint(-3, P + 3, (L,), generator=g, dtype=torch.int64)
        pos[: min(L, 4)] = pos[0]
    dH = (torch.randn((B, L, C_), generator=g) * torch.exp(torch.randn((B, L, 1), generator=g))).to(torch.bfloat16)
    dtok0 = torch.randn((V, C_), generator=g) * 0.5
    dpos0 = torch.randn((P, C_), generator=g) * 0.5
    return ids, pos, dH, dtok0, dpos0


def run_kernel(ids, pos, dH, dtok0, dpos0, V, P, want_tok=True, want_pos=True):
    dtok = dtok0.to(DEV).clone() if want_tok else None
    dpos = dpos0.to(DEV).clone() if want_pos else None
    rc = call_grad(ids.to(DEV), None if pos is None else pos.to(DEV), dH.to(DEV), dtok, dpos, V, P)
    assert rc == 0, _lib.lib().hcp_last_error_string().decode()
    torch.cuda.synchronize()
    return (None if dtok is None else dtok.cpu()), (None if dpos is None else dpos.cpu())


@pytest.mark.parametrize("case", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_embed_grad_bit_exact_and_within_fp64_bound(case):
    name, B, L, C_, V, P, _, _ = case
    ids, pos, dH, dtok0, dpos0 = kernel_inputs(case)
    got_tok, got_pos = run_kernel(ids, pos, dH, dtok0, dpos0, V, P)
    ktok, kpos = keys_of(ids.numpy(), None if pos is None else pos.numpy(), V, P)
    dh = dH.float().reshape(B * L, C_).numpy()
    worst = 0.0
    for got, keys, d0 in ((got_tok, ktok, dtok0), (got_pos, kpos, dpos0)):
        want, want64, mag, cnt = restate(keys, dh, d0.numpy())
        assert np.array_equal(got.numpy().view(np.uint32), want.view(np.uint32)), f"{name}: differs from the documented order"
        bound = (cnt[:, None] + 1) * 2.0 ** -24 * mag
        err = np.abs(got.numpy().astype(np.float64) - want64)
        assert (err <= bound).all(), f"{name}: beyond the fp32 sum bound"
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
        untouched = np.setdiff1d(np.arange(d0.shape[0]), keys)
        assert np.array_equal(got.numpy()[untouched], d0.numpy()[untouched])
    print(f"[embed_grad {name}] worst error / bound {worst:.3f}")


@pytest.mark.parametrize("which", ["tok_only", "pos_only"])
def test_embed_grad_one_destination(which):
    case = KERNEL_CASES[2]
    _, B, L, C_, V, P, _, _ = case
    ids, pos, dH, dtok0, dpos0 = kernel_inputs(case, seed=3)
    both_tok, both_pos = run_kernel(ids, pos, dH, dtok0, dpos0, V, P)
    tok, posg = run_kernel(ids, pos, dH, dtok0, dpos0, V, P, want_tok=which == "tok_only", want_pos=which == "pos_only")
    if which == "tok_only":
        assert posg is None and torch.equal(tok, both_tok)
    else:
        assert tok is None and torch.equal(posg, both_pos)


def test_embed_grad_repeats_and_graph_are_bit_identical():
    case = KERNEL_CASES[2]
    _, B, L, C_, V, P, _, _ = case
    ids, pos, dH, dtok0, dpos0 = (t.to(DEV) if t is not None else None for t in kernel_inputs(case, seed=5))
    nbytes = _lib.lib().hcp_embed_grad_workspace_bytes(B, L, C_)
    ws = torch.empty(((nbytes + 15) // 16 * 4,), dtype=torch.float32, device=DEV)
    outs = []
    for _ in range(3):
        dtok, dpos = dtok0.clone(), dpos0.clone()
        assert call_grad(ids, pos, dH, dtok, dpos, V, P, ws) == 0
        outs.append((dtok, dpos))
    dtok_g, dpos_g = dtok0.clone(), dpos0.clone()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        assert call_grad(ids, pos, dH, dtok_g, dpos_g, V, P, ws) == 0
    graph.replay()
    torch.cuda.synchronize()
    for dtok, dpos in outs[1:] + [(dtok_g, dpos_g)]:
        assert torch.equal(dtok, outs[0][0]) and torch.equal(dpos, outs[0][1])


def test_embed_grad_refusals():
    B, L, C_, V, P = 2, 77, 64, 100, 77
    ids = torch.randint(0, V, (B, L), device=DEV)
    dH = torch.randn((B, L, C_), device=DEV).to(torch.bfloat16)
    dtok, dpos = torch.full((V, C_), 0.25, device=DEV), torch.full((P, C_), 0.25, device=DEV)
    nbytes = _lib.lib().hcp_embed_grad_workspace_bytes(B, L, C_)
    assert nbytes > 0 and _lib.lib().hcp_embed_grad_workspace_bytes(0, L, C_) == 0
    ws = torch.zeros(((nbytes + 15) // 16 * 4 + 4,), dtype=torch.float32, device=DEV)
    f = _lib.lib().hcp_embed_grad_bf16
    big = torch.zeros(2 * L, dtype=torch.int64, device=DEV)
    ok = dict(ids=ids.data_ptr(), pos=None, dH=dH.data_ptr(), B=B, L=L, C=C_, dtok=dtok.data_ptr(), V=V, dpos=dpos.data_ptr(), P=P,
              ws=ws.data_ptr(), wsb=nbytes)
    bad = [dict(ids=None), dict(dH=None), dict(ws=None), dict(dtok=None, dpos=None), dict(B=0), dict(L=0), dict(C=0), dict(C=-8),
           dict(C=12), dict(V=0), dict(P=0), dict(B=-1), dict(L=P + 1, ids=big.data_ptr()), dict(dH=dH.data_ptr() + 2),
           dict(dtok=dtok.data_ptr() + 4), dict(dpos=dpos.data_ptr() + 8), dict(ws=ws.data_ptr() + 4), dict(ids=ids.data_ptr() + 4),
           dict(wsb=nbytes - 1), dict(V=1 << 31)]
    before = _lib.launch_count
    for change in bad:
        a = {**ok, **change}
        rc = f(a["ids"], a["pos"], a["dH"], a["B"], a["L"], a["C"], a["dtok"], a["V"], a["dpos"], a["P"], a["ws"], a["wsb"], stream_ptr())
        assert rc == -1, change                                  # HCP_ERR_INVALID
    assert _lib.launch_count == before
    torch.cuda.synchronize()
    assert bool((dtok == 0.25).all()) and bool((dpos == 0.25).all())
    # L > P is fine once the positions are given (or when only the token table is trained)
    big_h = torch.zeros((B, P + 1, C_), device=DEV, dtype=torch.bfloat16)
    ids2 = torch.zeros((B, P + 1), dtype=torch.int64, device=DEV)
    nb2 = _lib.lib().hcp_embed_grad_workspace_bytes(B, P + 1, C_)
    ws2 = torch.zeros(((nb2 + 15) // 16 * 4,), dtype=torch.float32, device=DEV)
    assert f(ids2.data_ptr(), None, big_h.data_ptr(), B, P + 1, C_, dtok.data_ptr(), V, None, P, ws2.data_ptr(), nb2, stream_ptr()) == 0


# ---------------------------------------------------------------------------------------------------------------------------------
# every parameter gradient
# ---------------------------------------------------------------------------------------------------------------------------------
def check_param_grads(model, ref_sd, name_map=lambda n: n, lora_pairs=()):
    """Every trainable parameter of `model` against the fp32 reference leaf of the same name; zero reference gradients are exact.
    The k_proj bias is the exception: softmax ignores a shift of every score of a query row, so its exact gradient is 0 and both sides
    hold rounding noise; its norm is held to 5e-2 of the same layer's v_proj bias gradient instead."""
    worst = []
    for name, p in model.named_parameters():
        if not p.requires_grad or "lora_block_" in name:
            continue
        ref_p = ref_sd[name_map(name)]
        ref = ref_p.grad
        got = p.grad
        if ref is None or float(ref.abs().max()) == 0.0:
            assert got is None or float(got.abs().max()) == 0.0, f"{name}: expected an exactly zero gradient"
            continue
        assert got is not None, name
        if name.endswith("k_proj.bias") or name.endswith("k_proj._host.bias"):
            scale = ref_sd[name_map(name).replace("k_proj", "v_proj")].grad.double().norm()
            e = float(got.detach().double().norm().cpu() / scale)
            worst.append((e, name))
            continue
        e = rel(got, ref)
        worst.append((e, name))
        if name.endswith("token_embedding.weight"):
            unused = (ref.abs().amax(1) == 0).cpu()
            assert bool(unused.any()) and float(got.detach().cpu()[unused].abs().max()) == 0.0, "unused token rows must be exactly 0"
    for name, got, ref in lora_pairs:
        e = rel(got, ref)
        worst.append((e, name))
    worst.sort(reverse=True)
    print("worst parameter gradients:", [(f"{e:.2e}", n) for e, n in worst[:5]])
    for e, n in worst:
        assert e <= 5e-2, (n, e)
    return worst


def te_with_full_ft(spec, sd, layers=("",), lora_layers=None):
    te = CLIPTextModel(**spec.kwargs())
    te.load_state_dict(sd)
    te = te.to(DEV).requires_grad_(False)
    lora_cfg = None if lora_layers is None else [{"rank": 4, "alpha": 1.0, "layers": list(lora_layers)}]
    groups, lgroup = make_hcpdiff(te, [{"lr": 1e-5, "layers": list(layers)}], lora_cfg)
    return te, groups, lgroup


@pytest.mark.parametrize("n_repeats,clip_skip,final_norm", [(1, 0, True), (2, 0, True), (1, 1, True), (1, 0, False), (2, 1, False)])
def test_tiny_te_every_parameter_gradient(n_repeats, clip_skip, final_norm):
    spec = R.TINY_TE
    sd = R.init_params(spec, seed=5)
    te, _, _ = te_with_full_ft(spec, sd)
    assert all(p.requires_grad for p in te.parameters())
    ids = R.synthetic_ids(3, n_repeats, seed=21)
    ehs = encode_prompt(te, ids.to(DEV), n_repeats, clip_skip, final_norm)
    G = torch.randn(ehs.shape, generator=torch.Generator().manual_seed(4))
    (ehs.float() * G.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ehs_r = R.encode_prompt(ref_sd, ids, spec, n_repeats, clip_skip, final_norm, training=True)
    assert rel(ehs, ehs_r) < 2e-2
    (ehs_r * G).sum().backward()
    check_param_grads(te, ref_sd)
    for i in range(spec.num_hidden_layers - clip_skip, spec.num_hidden_layers):      # the layers clip_skip cuts: exactly 0
        for n, p in te.text_model.encoder.layers[i].named_parameters():
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, n


def test_tiny_te_full_ft_and_lora_on_the_same_layers():
    """A layer both in `text_encoder:` and wrapped by `lora_text_encoder`: as in the UNet, its pack keeps the trained base weight
    (refreshed by repack_trained) and the LoRA factors as a separate GEMM segment, and both gradients are produced."""
    spec = R.TINY_TE
    sd = R.init_params(spec, seed=5)
    te, _, lgroup = te_with_full_ft(spec, sd, layers=["text_model.encoder.layers.0", "text_model.embeddings"],
                                    lora_layers=["re:.*self_attn$"])
    lora = {k: v for k, v in R.init_lora(spec, rank=4, up_std=0.05).items() if k in lgroup.plugin_dict}
    with torch.no_grad():
        for k, (e,) in lora.items():
            lgroup[k].layer.W_down.copy_(e.W_down)
            lgroup[k].layer.W_up.copy_(e.W_up)
            lgroup[k].layer.W_down.grad = lgroup[k].layer.W_up.grad = None
    ids = R.synthetic_ids(2, 1, seed=22)
    ehs = encode_prompt(te, ids.to(DEV), 1, 0, True)
    G = torch.randn(ehs.shape, generator=torch.Generator().manual_seed(6))
    (ehs.float() * G.to(DEV)).sum().backward()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref_lora = {k: [U.LoraEntry(e.W_down.clone().requires_grad_(True), e.W_up.clone().requires_grad_(True), e.alpha, None)]
                for k, (e,) in lora.items()}
    (R.encode_prompt(ref_sd, ids, spec, 1, 0, True, lora=ref_lora) * G).sum().backward()
    # base parameter names of a wrapped layer read `<layer>._host.weight` (the reference's container layout)
    pairs = []
    for k, (e,) in ref_lora.items():
        pairs += [(k + ".W_down", lgroup[k].layer.W_down.grad, e.W_down.grad), (k + ".W_up", lgroup[k].layer.W_up.grad, e.W_up.grad)]
    worst = check_param_grads(te, ref_sd, name_map=lambda n: n.replace("._host", ""), lora_pairs=pairs)
    assert any("_host" in n for _, n in worst)
    frozen = [n for n, p in te.named_parameters() if (".layers.1." in n or "final_layer_norm" in n) and "lora_block_" not in n]
    assert frozen and all(not p.requires_grad and p.grad is None for n, p in te.named_parameters() if n in frozen)


@pytest.mark.parametrize("clip_skip,final_norm", [(0, True), (1, False)])
def test_tiny_sdxl_pair_every_parameter_gradient(clip_skip, final_norm):
    pair = X.TINY_XL_TE
    sd = X.init_params(pair, seed=3)
    te = SDXLTextEncoder(**pair.kwargs())
    te.load_state_dict(sd)
    te = te.to(DEV).requires_grad_(False)
    make_hcpdiff(te, [{"lr": 1e-5, "layers": [""]}], None)
    assert te.clip_bigG.text_projection.weight.requires_grad
    ids = X.synthetic_ids(3, seed=9)
    ehs, emb = encode_prompt_sdxl(te, ids.to(DEV), clip_skip, final_norm)
    g = torch.Generator().manual_seed(8)
    G1, G2 = torch.randn(ehs.shape, generator=g), torch.randn(emb.shape, generator=g)
    ((ehs.float() * G1.to(DEV)).sum() + (emb.float() * G2.to(DEV)).sum()).backward()
    ref_sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ehs_r, emb_r = X.encode_prompt_sdxl(ref_sd, ids, pair, clip_skip, final_norm, training=True)
    ((ehs_r * G1).sum() + (emb_r * G2).sum()).backward()
    worst = check_param_grads(te, ref_sd)
    assert any(n == "clip_bigG.text_projection.weight" for _, n in worst)


# ---------------------------------------------------------------------------------------------------------------------------------
# joint steps with the UNet
# ---------------------------------------------------------------------------------------------------------------------------------
AF_KW = {"lr": 1e-4, "relative_step": False, "weight_decay": 1e-3}
TE_OPTS = {"n_repeats": 1, "clip_skip": 1, "clip_final_norm": True}


def joint_reference(unet_sd, unet_lora, unet_names, te_sd, te_names, optimizer, lr, te_lr, max_norm):
    """clip_ref.joint_reference_loop with the text encoder's base tensors as the trained leaves (one more param group)."""
    spec, tspec = U.TINY, R.TINY_TE

    class Joint(S.ReferenceLoop):
        def __init__(self):
            super().__init__(unet_sd, unet_lora, spec, lr=lr, max_grad_norm=max_norm, train_base=unet_names)
            leaves = [te_sd[n].requires_grad_(True) for n in te_names]
            self.opt.add_param_group({"params": leaves, "lr": te_lr})
            self.leaves += leaves
            if optimizer == "adafactor":
                kw = {k: v for k, v in AF_KW.items() if k != "lr"}
                self.opt = AF.OracleAdafactor([{"params": g["params"], "lr": g["lr"]} for g in self.opt.param_groups], **kw)

        def micro_step(self, latents, noise, t, ids):
            ehs = R.encode_prompt(te_sd, ids, tspec, training=True, **TE_OPTS)
            return super().micro_step(latents, noise, t, ehs)

    return Joint()


def update_check(label, got, want):
    cos = float(got.double() @ want.double() / (got.double().norm() * want.double().norm()))
    ratio = float(got.norm() / want.norm())
    print(f"[{label}] update cos {cos:.4f} norm ratio {ratio:.4f}")
    assert cos >= 0.9 and 0.9 < ratio < 1.1, label


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("optimizer", ["adamw", "adafactor"])
@pytest.mark.parametrize("unet_mode", ["lora", "full"])
def test_joint_unet_and_te_full_ft_steps_match_reference_loop(unet_mode, optimizer, use_graph):
    spec, tspec = U.TINY, R.TINY_TE
    sd = U.init_params(spec)
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    lr = 1e-4 if unet_mode == "lora" else 1e-5
    if unet_mode == "lora":
        ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": lr, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
        lora = U.init_lora(spec, rank=4)
        with torch.no_grad():
            for layer, entries in lora.items():
                ugroup[layer].layer.W_down.copy_(entries[0].W_down)
                ugroup[layer].layer.W_up.copy_(entries[0].W_up)
        unet_names, unet_prod = [], [p for b in ugroup.plugin_dict.values() for p in (b.layer.W_down, b.layer.W_up)]
        unet_ref_leaves = [p for k in ugroup.plugin_dict for p in (lora[k][0].W_down, lora[k][0].W_up)]
    else:
        ugroups, _ = make_hcpdiff(unet, [{"lr": lr, "layers": [""]}], None)
        lora = None
        unet_names = [n for n, _ in unet.named_parameters()]
        unet_prod = [p for _, p in unet.named_parameters()]
        ref_usd = {k: v.clone() for k, v in sd.items()}
    tsd = R.init_params(tspec, seed=5)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    te_lr = 1e-5
    tgroups, _ = make_hcpdiff(te, [{"lr": te_lr, "layers": [""]}], None, default_lr=1e-5)
    te_names = [n for n, _ in te.named_parameters()]
    ref_tsd = {k: v.clone() for k, v in tsd.items()}
    usd_for_ref = sd if unet_mode == "lora" else ref_usd
    ref = joint_reference(usd_for_ref, lora, unet_names, ref_tsd, te_names, optimizer, lr, te_lr, 1.0)
    if unet_mode == "full":
        unet_ref_leaves = [ref_usd[n] for n in unet_names]
    kw = {"optimizer_kwargs": AF_KW} if optimizer == "adafactor" else {}
    step = LoraTrainStep(unet, ugroups + tgroups, lr=lr, max_grad_norm=1.0, use_cuda_graph=use_graph, optimizer=optimizer,
                         text_encoder=te, text_encoder_opts=TE_OPTS, **kw)
    u0 = [p.detach().clone() for p in unet_prod]
    ur0 = [p.detach().clone() for p in unet_ref_leaves]
    t0 = {n: p.detach().clone() for n, p in te.named_parameters()}
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, spec, seed=100 + i)
        ids = R.synthetic_ids(2, 1, seed=200 + i)
        loss = float(step.step(lat, noise, t, ids).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids)
        print(f"[joint {unet_mode} {optimizer} graph={use_graph} step {i}] loss {loss:.6f} ref {loss_ref:.6f}")
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref)
    label = f"{unet_mode} {optimizer} graph={use_graph}"
    update_check(label + " unet", torch.cat([(p.detach() - q).flatten().cpu() for p, q in zip(unet_prod, u0)]),
                 torch.cat([(p.detach() - q).flatten() for p, q in zip(unet_ref_leaves, ur0)]))
    update_check(label + " te", torch.cat([(p.detach() - t0[n]).flatten().cpu() for n, p in te.named_parameters()]),
                 torch.cat([(ref_tsd[n].detach() - tsd[n]).flatten() for n in te_names]))


# ---------------------------------------------------------------------------------------------------------------------------------
# the entry point
# ---------------------------------------------------------------------------------------------------------------------------------
def test_train_ac_dreambooth_te_config_saves_resumes_and_logs_group_losses(tmp_path):
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    with open(os.path.join(ROOT, "cfgs/train/dreambooth_te_sd15_synthetic.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["exp_dir"] = os.path.join(tmp_path, "exp")
    cfg["model"]["unet"].update(sample_size=16, block_out_channels=[64, 128, 128, 128], attention_head_dim=2, cross_attention_dim=64)
    cfg["model"]["text_encoder"] = {"_target_": "hcp_diffusion_b200.models.CLIPTextModel", **R.TINY_TE.kwargs()}
    cfg["model"]["ema"] = {"decay_max": 0.99}
    cfg["train"].update(train_steps=2, save_step=2, log_step=1)
    cfg["train"]["scheduler"]["num_warmup_steps"] = 1                  # the warm-up's first step has lr 0; the second one trains
    for g in cfg["data"].values():
        g["num_samples"] = 8
    path = os.path.join(tmp_path, "te_ft.yaml")
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", path], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "step 2/2" in r.stdout
    ck = os.path.join(tmp_path, "exp", "ckpts", "text_encoder-2.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert set(sd) == {"base", "base_ema"}
    assert set(sd["base"]) == set(R.param_shapes(R.TINY_TE)) == set(sd["base_ema"])     # transformers' names, every tensor
    shapes = R.param_shapes(R.TINY_TE)
    assert all(tuple(v.shape) == shapes[k] for k, v in sd["base"].items())
    assert any(not torch.equal(sd["base"][k], sd["base_ema"][k]) for k in sd["base"])
    uck = os.path.join(tmp_path, "exp", "ckpts", "unet-2.safetensors")
    conf = load_config_with_cli(path, [f"train.resume.ckpt_path.TE=[{ck}]", f"train.resume.ckpt_path.unet=[{uck}]",
                                       "train.resume.start_step=2", "train.train_steps=3"])
    tr = Trainer(conf)
    live = dict(tr.te.named_parameters())
    for k, v in sd["base"].items():
        assert torch.equal(live[k].detach().cpu(), v), k
    assert tr.step_fn.flat.numel >= sum(v.numel() for v in sd["base"].values())
    tr.train()
    assert all(math.isfinite(v) and v > 0 for v in tr.step_fn.loss.cpu().tolist())      # one loss per data group
