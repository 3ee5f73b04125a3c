"""GPU parity tests (run with `pytest -m gpu` on an H100): the CUDA path, called through the C ABI, against
  * plain fp32 PyTorch references of each op (same inputs, bf16-rounded where the kernel rounds),
  * the golden vectors generated from the real reference LoRA classes (tests/golden/ref_lora_linear.pt),
  * the CPU oracle (oracle/unet_ref.py) on the TINY topology and on full-size SD1.5.

Tolerances (stated per SURVEY.md 8d): the kernels compute in bf16 with fp32 accumulation, the oracle in fp32 --
  per-op relative L2 <= 1e-2;  end-to-end noise_pred relative L2 <= 2e-2 and max-abs <= 5e-2 * max|ref|;
  LoRA gradients relative L2 <= 5e-2 (they pass through ~60 bf16 layers twice).
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import ops  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import LoraLayer, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.ops import ConvPack, LinearPack, LoraBlockRef  # noqa: E402
from hcp_diffusion_b200.runtime import pack_lora  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16


def rel_l2(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def bf(x):
    return x.to(BF).float()


# ----------------------------------------------------------------------------------------------------------------------
# per-op parity against fp32 torch
# ----------------------------------------------------------------------------------------------------------------------
# last rows: the benchmark's dominant GEMM shapes (config 2, batch 4): ff.net.0.proj at 64x64 (M 16384, K 320, N 2560), the fused QKV with
# three rank-8 blocks at 64x64, and the K = 10240 split-K linear of the 16x16 level
@pytest.mark.parametrize("M,K,N,ranks", [(256, 320, 320, (8,)), (77, 768, 640, (8, 8)), (1024, 320, 960, (8, 8, 8)), (64, 1280, 1280, ()),
                                         (16384, 320, 2560, ()), (16384, 320, 960, (8, 8, 8)), (1024, 10240, 1280, ()), (256, 1280, 1280, (8,))])
@pytest.mark.parametrize("merge,tiled", [(False, False), (True, False), (True, True), (False, True)])
def test_linear_lora_fwd_bwd(M, K, N, ranks, merge, tiled):
    """merge=False: the LoRA delta as an extra K-segment of the GEMM; merge=True: adapters merged into the bf16 operands per step
    (hcp_lora_merge), plain GEMMs forward / dgrad, T and U only for the factor gradients."""
    if merge and not ranks:
        pytest.skip("nothing to merge")
    if tiled and (K % 64 or N % 64):
        pytest.skip("k-block-major operands need 64-element multiples")
    x = rnd(M, K, seed=1).to(BF).requires_grad_(True)
    W = rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    b = rnd(N, scale=0.1, seed=3)
    res = rnd(M, N, seed=4).to(BF).requires_grad_(True)
    pack = LinearPack(W, b)
    if tiled:
        pack.tile_weights()
        assert pack.tiled
    blocks, refs, c0 = [], [], 0
    n_per = N // max(len(ranks), 1)
    for i, r in enumerate(ranks):          # block i patches output rows [i*n_per, (i+1)*n_per): the fused-QKV arrangement
        down = rnd(r, K, scale=1 / math.sqrt(K), seed=10 + i).requires_grad_(True)
        up = rnd(n_per, r, scale=0.3, seed=20 + i).requires_grad_(True)
        blocks.append((down, up, 0.125))
        refs.append(LoraBlockRef(down, up, 0.125, i * n_per))
        c0 += r
    if refs:
        pack.attach_lora(refs)
        if merge:
            assert pack.enable_merge([(W[i * n_per:(i + 1) * n_per], i * n_per, n_per, [ref]) for i, ref in enumerate(refs)])

        class G:
            pass
        g = G()
        g.pack = pack
        pack_lora([g])
    y = ops.fused_linear(pack, [x], residual=res)
    # reference: materialised W' like the reference operator, on bf16-rounded operands
    Wf = bf(W).clone()
    xr = x.detach().float().requires_grad_(True)
    rr = res.detach().float().requires_grad_(True)
    dl = [(d.detach().clone().requires_grad_(True), u.detach().clone().requires_grad_(True)) for d, u, _ in blocks]
    Wp = Wf
    if dl:
        delta = torch.zeros_like(Wf)
        for i, (d, u) in enumerate(dl):
            delta[i * n_per:(i + 1) * n_per] = 0.125 * (u @ d)
        Wp = Wf + delta
    yr = xr @ Wp.t() + b + rr
    assert rel_l2(y, yr) < 1e-2
    dy = rnd(M, N, seed=5).to(BF)
    y.backward(dy)
    yr.backward(dy.float())
    assert rel_l2(x.grad, xr.grad) < 1e-2
    torch.testing.assert_close(res.grad.float(), dy.float())
    for (d, u, _), (dr, ur) in zip(blocks, dl):
        assert rel_l2(d.grad, dr.grad) < 2e-2
        assert rel_l2(u.grad, ur.grad) < 2e-2


def test_reference_lora_golden_through_product_container(golden_dir):
    """The vectors the REAL reference LoraLayer/LoraPatchContainer produced (fp32) vs the product container on the GPU."""
    fx = torch.load(os.path.join(golden_dir, "ref_lora_linear.pt"))

    class Attn(torch.nn.Module):
        def __init__(self, c, ctx):
            super().__init__()
            self.to_q = torch.nn.Linear(c, c, bias=False)
            self.to_k = torch.nn.Linear(ctx, c, bias=False)
            self.to_out = torch.nn.ModuleList([torch.nn.Linear(c, c, bias=True), torch.nn.Dropout(0.0)])

    class Blk(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.attn1, self.attn2 = Attn(48, 48), Attn(48, 24)

    model = Blk()
    model.load_state_dict({k.replace("._host", ""): v for k, v in fx["host"].items()})
    model = model.to(DEV).requires_grad_(False)
    named = dict(model.named_modules())
    blocks = {}
    for lname in ("attn1", "attn2"):
        d = LoraLayer.wrap_model(0, named[lname], parent_block=None, host_name=None, rank=4, dropout=0.0, alpha=1.0)
        blocks.update({f"{lname}.{k}": v for k, v in d.items()})
    second = LoraLayer.wrap_model(1, model.attn1.to_q, parent_block=model.attn1, host_name="to_q", rank=2, dropout=0.0, alpha=0.5)[""]
    with torch.no_grad():
        for path, blk in blocks.items():
            blk.layer.W_down.copy_(fx["ckpt"][f"{path}.___.layer.W_down"])
            blk.layer.W_up.copy_(fx["ckpt"][f"{path}.___.layer.W_up"])
            assert abs(float(blk.alpha) - float(fx["ckpt"][f"{path}.___.alpha"])) < 1e-7
        second.layer.W_down.copy_(fx["second_block"]["layer.W_down"])
        second.layer.W_up.copy_(fx["second_block"]["layer.W_up"])
    assert sorted(model.state_dict().keys()) == fx["state_keys_model"]
    x = fx["x"].to(DEV).requires_grad_(True)
    ctx = fx["ctx"].to(DEV)
    outs = {"attn1.to_q": model.attn1.to_q(x), "attn1.to_k": model.attn1.to_k(x), "attn1.to_out.0": model.attn1.to_out[0](x),
            "attn2.to_k": model.attn2.to_k(ctx), "attn2.to_q": model.attn2.to_q(x)}
    for k, v in outs.items():
        assert v.dtype == torch.float32 and rel_l2(v, fx["outs"][k]) < 1e-2, k
    sum((o ** 2).sum() for o in outs.values()).backward()
    assert rel_l2(x.grad, fx["grad_x"]) < 2e-2
    for name, p in model.named_parameters():
        if "lora_block" in name and name in fx["grads"]:          # layers the golden loss did not touch have no gradient
            assert rel_l2(p.grad, fx["grads"][name]) < 3e-2, name
    assert sum(1 for n, _ in model.named_parameters() if n in fx["grads"]) == len(fx["grads"])


# last rows: the benchmark's dominant convolutions (config 2, batch 4): 960->320 at 64x64 (two M tiles per work item), 1280->1280 at 16x16
# and 8x8 (split-K), 320->320 at 64x64 and the stride-2 downsampler
@pytest.mark.parametrize("B,H,W,Cin,Cout,stride", [(2, 16, 16, 64, 128, 1), (2, 32, 32, 320, 320, 2), (3, 8, 8, 128, 64, 1), (1, 64, 64, 64, 64, 1),
                                                   (4, 64, 64, 960, 320, 1), (4, 16, 16, 1280, 1280, 1), (4, 8, 8, 1280, 1280, 1),
                                                   (4, 64, 64, 320, 320, 1), (4, 64, 64, 320, 320, 2), (4, 8, 8, 2560, 1280, 1)])
@pytest.mark.parametrize("tiled", [False, True])
def test_conv3x3_fwd_bwd(B, H, W, Cin, Cout, stride, tiled):
    """tiled: k-block-major weight operands ([9*C/64][rows][64], hcp_conv3x3_args.w_tiled) for the forward and the dgrad."""
    if tiled and (Cin % 64 or Cout % 64):
        pytest.skip("k-block-major operands need 64-channel multiples")
    x = rnd(B, H * W, Cin, seed=1).to(BF).requires_grad_(True)
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2)
    b = rnd(Cout, scale=0.1, seed=3)
    rb = rnd(B, Cout + 8, scale=0.5, seed=4)[:, 4:4 + Cout]          # a strided view, like the time-embedding slices
    Ho, Wo = H // stride, W // stride
    res = rnd(B, Ho * Wo, Cout, seed=5).to(BF).requires_grad_(True)
    pack = ConvPack(w, b, stride)
    if tiled:
        pack.tile_weights()
        assert pack.tiled
    y = ops.conv3x3(pack, x, (B, H, W), rowbias=rb, residual=res)
    xr = x.detach().float().view(B, H, W, Cin).permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.conv2d(xr, bf(w), b, stride=stride, padding=1) + rb[:, :, None, None] + res.detach().float().view(B, Ho, Wo, Cout).permute(0, 3, 1, 2)
    yr_nhwc = yr.permute(0, 2, 3, 1).reshape(B, Ho * Wo, Cout)
    assert rel_l2(y, yr_nhwc) < 1e-2
    dy = rnd(B, Ho * Wo, Cout, seed=6).to(BF)
    y.backward(dy)
    yr_nhwc.backward(dy.float())
    assert rel_l2(x.grad, xr.grad.permute(0, 2, 3, 1).reshape(B, H * W, Cin)) < 1e-2
    torch.testing.assert_close(res.grad.float(), dy.float())


@pytest.mark.parametrize("B,HW,C1,C2,silu,eps", [(2, 256, 320, 0, True, 1e-5), (2, 64, 1280, 640, True, 1e-5), (3, 1024, 640, 0, False, 1e-6), (1, 4096, 640, 320, True, 1e-5)])
def test_groupnorm_fwd_bwd(B, HW, C1, C2, silu, eps):
    C = C1 + C2
    x1 = (rnd(B, HW, C1, seed=1) * 2 + 0.5).to(BF).requires_grad_(True)
    x2 = (rnd(B, HW, C2, seed=2) - 0.3).to(BF).requires_grad_(True) if C2 else None
    gamma = 1 + 0.1 * rnd(C, seed=3)
    beta = 0.1 * rnd(C, seed=4)
    outs = ops.group_norm(gamma, beta, 32, eps, silu, x1, x2)
    y = outs[0]
    xr = torch.cat([x1.detach().float()] + ([x2.detach().float()] if C2 else []), -1).requires_grad_(True)
    yr = F.group_norm(xr.transpose(1, 2), 32, gamma, beta, eps)
    yr = (F.silu(yr) if silu else yr).transpose(1, 2)
    assert rel_l2(y, yr) < 1e-2
    dy = rnd(B, HW, C, seed=5).to(BF)
    d1 = rnd(B, HW, C1, seed=6).to(BF)
    loss = (y.float() * dy.float()).sum() + (outs[1].float() * d1.float()).sum()
    loss.backward()
    yr.backward(dy.float())
    assert rel_l2(x1.grad, xr.grad[..., :C1] + d1.float()) < 1e-2
    if C2:
        assert rel_l2(x2.grad, xr.grad[..., C1:]) < 1e-2


@pytest.mark.parametrize("M,C", [(512, 320), (300, 640), (64, 1280)])
def test_layernorm_fwd_bwd(M, C):
    x = (rnd(M, C, seed=1) * 1.5 + 0.2).to(BF).requires_grad_(True)
    gamma, beta = 1 + 0.1 * rnd(C, seed=2), 0.1 * rnd(C, seed=3)
    y, alias = ops.layer_norm(gamma, beta, 1e-5, x)
    xr = x.detach().float().requires_grad_(True)
    yr = F.layer_norm(xr, (C,), gamma, beta, 1e-5)
    assert rel_l2(y, yr) < 1e-2
    dy, da = rnd(M, C, seed=4).to(BF), rnd(M, C, seed=5).to(BF)
    ((y.float() * dy.float()).sum() + (alias.float() * da.float()).sum()).backward()
    yr.backward(dy.float())
    assert rel_l2(x.grad, xr.grad + da.float()) < 1e-2


def test_geglu_and_upsample():
    u = rnd(300, 2 * 640, seed=1).to(BF).requires_grad_(True)
    h = ops.GegluFn.apply(u)
    ur = u.detach().float().requires_grad_(True)
    a, g = ur.chunk(2, -1)
    hr = a * F.gelu(g)
    assert rel_l2(h, hr) < 1e-2
    dh = rnd(300, 640, seed=2).to(BF)
    h.backward(dh)
    hr.backward(dh.float())
    assert rel_l2(u.grad, ur.grad) < 1e-2
    x = rnd(2, 8 * 8, 64, seed=3).to(BF).requires_grad_(True)
    y = ops.Upsample2xFn.apply((2, 8, 8), x)
    xr = x.detach().float().view(2, 8, 8, 64).permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.interpolate(xr, scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1).reshape(2, 256, 64)
    torch.testing.assert_close(y.float(), yr)
    dy = rnd(2, 256, 64, seed=4).to(BF)
    y.backward(dy)
    yr.backward(dy.float())
    assert rel_l2(x.grad, xr.grad.permute(0, 2, 3, 1).reshape(2, 64, 64)) < 1e-2


# last rows: the benchmark's attention shapes (config 2, batch 4): self-attention L = 4096, d = 40 (87 % of the attention FLOPs) and its
# cross-attention twin against 77 text tokens
@pytest.mark.parametrize("B,H,L,Lkv,d,mask", [(2, 8, 256, 256, 40, False), (2, 8, 200, 77, 40, True), (1, 8, 1024, 1024, 80, False), (2, 8, 64, 64, 160, False), (2, 8, 256, 77, 160, True),
                                              (4, 8, 4096, 4096, 40, False), (4, 8, 4096, 77, 40, False), (4, 8, 1024, 1024, 80, False)])
def test_attention_fwd_bwd(B, H, L, Lkv, d, mask):
    C = H * d
    self_attn = (L == Lkv) and not mask
    if self_attn:
        qkv = rnd(B, L, 3 * C, scale=1.0, seed=1).to(BF).requires_grad_(True)
        o = ops.attention(H, C, (0, C, 2 * C), qkv)
        q, k, v = qkv.detach().float().split(C, -1)
        kv_bias = None
    else:
        qs = rnd(B, L, C, seed=1).to(BF).requires_grad_(True)
        kvs = rnd(B, Lkv, 2 * C, seed=2).to(BF).requires_grad_(True)
        kv_bias = None
        if mask:
            m = torch.ones(B, Lkv, device=DEV)
            m[:, -5:] = 0
            kv_bias = (1 - m) * -10000.0
        o = ops.attention(H, C, (0, 0, C), qs, kvs, kv_bias)
        q = qs.detach().float()
        k, v = kvs.detach().float().split(C, -1)
    q, k, v = (t.clone().requires_grad_(True) for t in (q, k, v))
    qh, kh, vh = (t.view(B, -1, H, d).transpose(1, 2) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / math.sqrt(d)
    if kv_bias is not None:
        s = s + kv_bias[:, None, None, :]
    orf = (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, L, C)
    assert rel_l2(o, orf) < 1e-2
    do = rnd(B, L, C, seed=3).to(BF)
    o.backward(do)
    orf.backward(do.float())
    if self_attn:
        ref = torch.cat([q.grad, k.grad, v.grad], -1)
        assert rel_l2(qkv.grad, ref) < 2e-2
    else:
        assert rel_l2(qs.grad, q.grad) < 2e-2
        assert rel_l2(kvs.grad, torch.cat([k.grad, v.grad], -1)) < 2e-2


# ----------------------------------------------------------------------------------------------------------------------
# end to end against the CPU oracle
# ----------------------------------------------------------------------------------------------------------------------
def build_product_unet(spec, sd, lora_rank=0, lora_seed=1):
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    lora_oracle, group = None, None
    if lora_rank:
        groups, group = make_hcpdiff(unet, None, [{"rank": lora_rank, "alpha": 1.0, "dropout": 0.0, "layers": [r"re:.*\.attn.?$"]}])
        lora_oracle = U.init_lora(spec, rank=lora_rank, seed=lora_seed)
        with torch.no_grad():
            for layer, entries in lora_oracle.items():
                blk = group[layer]
                blk.layer.W_down.copy_(entries[0].W_down)
                blk.layer.W_up.copy_(entries[0].W_up)
                assert abs(float(blk.alpha) - entries[0].alpha) < 1e-7
        assert set(lora_oracle) == set(group.plugin_dict)
    return unet, group, lora_oracle


def check_end_to_end(spec, batch, rank, ctx_len, tol_pred=2e-2, tol_grad=5e-2):
    sd = U.init_params(spec)
    unet, group, lora_oracle = build_product_unet(spec, sd, rank)
    lat, noise, t, ehs = U.synthetic_batch(batch, spec, ctx_len=ctx_len)
    acp = U.ddpm_alphas_cumprod()
    x_t = U.add_noise(lat, noise, t, acp)
    if rank:
        loss_ref, pred_ref, grads_ref = U.lora_step_loss_and_grads(sd, lora_oracle, lat, noise, t, ehs, spec)
    else:
        with torch.no_grad():
            pred_ref = U.unet_forward(sd, x_t, t, ehs, spec=spec)
    pred = unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV)).sample
    assert pred.dtype == torch.float32 and pred.shape == pred_ref.shape
    err = rel_l2(pred, pred_ref)
    maxabs = float((pred.cpu() - pred_ref).abs().max() / pred_ref.abs().max())
    print(f"[{spec.block_out_channels} B={batch} r={rank}] noise_pred relL2={err:.3e} max-abs/max|ref|={maxabs:.3e}")
    assert err < tol_pred and maxabs < 5e-2
    if rank:
        loss = F.mse_loss(pred, noise.to(DEV), reduction="none").mean()
        assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
        loss.backward()
        num, den, worst = 0.0, 0.0, 0.0
        for layer, blocks in grads_ref.items():
            blk = group[layer]
            for got, ref in ((blk.layer.W_down.grad, blocks[0][0]), (blk.layer.W_up.grad, blocks[0][1])):
                num += float((got.cpu().double() - ref.double()).pow(2).sum())
                den += float(ref.double().pow(2).sum())
                worst = max(worst, rel_l2(got, ref))
        total = math.sqrt(num / den)
        print(f"    LoRA grads: global relL2={total:.3e}, worst layer relL2={worst:.3e}")
        assert total < tol_grad
    return unet


def test_tiny_unet_forward_no_lora():
    check_end_to_end(U.TINY, batch=2, rank=0, ctx_len=77)


@pytest.mark.parametrize("merge", [True, False])
def test_tiny_unet_lora_forward_backward(merge, monkeypatch):
    monkeypatch.setattr(ops, "LORA_MERGE", merge)
    check_end_to_end(U.TINY, batch=3, rank=4, ctx_len=77)


def test_sd15_forward_config1():
    """BASELINE.json configs[0]: SD1.5 UNet single forward, 1x4x64x64 latent, no LoRA."""
    check_end_to_end(U.SD15, batch=1, rank=0, ctx_len=77)


def test_sd15_lora_r8_forward_backward():
    """configs[1] topology and LoRA placement (rank 8 on every attn1/attn2 Linear) at B=1: noise_pred, loss and all 256 LoRA
    gradients against the fp32 oracle."""
    check_end_to_end(U.SD15, batch=1, rank=8, ctx_len=77)


def test_batch_invariance_and_zero_lora_identity():
    """Size-independent properties at the benchmark shape.  (1) Repeating a call is bit-exact (the forward has no
    floating-point atomics).  (2) An image gets the same result alone or inside a batch of 4 -- up to the summation order of
    split-K, whose plan depends on the launch size; measured 1.3e-2 -- two equally valid bf16 evaluations differ by about as
    much as either differs from the fp32 oracle -- so the bound is the oracle tolerance 2e-2, not bit equality.
    (3) A LoRA whose W_up is zero (the reference initialisation) reproduces the base model to the same tolerance."""
    sd = U.init_params(U.SD15)
    unet, group, _ = build_product_unet(U.SD15, sd, 0)
    lat, noise, t, ehs = U.synthetic_batch(4, U.SD15)
    x = lat.to(DEV)
    with torch.no_grad():
        full = unet(x, t.to(DEV), ehs.to(DEV)).sample
        again = unet(x, t.to(DEV), ehs.to(DEV)).sample
        assert torch.equal(full, again)
        one = unet(x[2:3], t[2:3].to(DEV), ehs[2:3].to(DEV)).sample
        assert rel_l2(one, full[2:3]) < 2e-2
        _, group = make_hcpdiff(unet, None, [{"rank": 8, "layers": [r"re:.*\.attn.?$"]}])     # reference init: W_up == 0
        with_lora = unet(x, t.to(DEV), ehs.to(DEV)).sample
        assert rel_l2(with_lora, full) < 2e-2        # mathematically identical; the extra K-segment may move a split-K boundary


def test_train_step_graph_matches_eager_and_learns():
    spec = U.TINY
    sd = U.init_params(spec)
    lat, noise, t, ehs = U.synthetic_batch(4, spec)
    results = []
    # eager single stream (the plain autograd order) vs eager / captured with the side stream (LoRA-gradient kernels and the
    # text-embedding k/v projections run concurrently with the main chain and are joined before the optimizer)
    for use_graph, side in ((False, False), (False, True), (True, True)):
        unet, group, _ = build_product_unet(spec, sd, 4)
        params = [p for b in group.plugin_dict.values() for p in b.parameters()]
        step = LoraTrainStep(unet, params, lr=1e-3, use_cuda_graph=use_graph, side_stream=side)
        losses = [float(step.step(lat, noise, t, ehs).cpu()) for _ in range(6)]
        results.append((losses, step.flat.data.clone()))
    (l0, p0), (l1, p1), (l2, p2) = results
    assert l0[-1] < l0[0]
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 1e-3 * abs(l0[0]) and max(abs(a - b) for a, b in zip(l0, l2)) < 1e-3 * abs(l0[0])
    assert rel_l2(p1, p0) < 1e-3 and rel_l2(p2, p0) < 1e-3


def test_reference_dapp_and_conv1x1_lora_golden_through_product_containers(golden_dir):
    """DreamArtist++ containers (batch = [negative | positive]) and LoRA on a 1x1 Conv2d: vectors of the REAL reference classes
    (tests/golden/ref_lora_dapp_conv.pt) vs the product containers on the GPU (bf16 operands, fp32 accumulate)."""
    from hcp_diffusion_b200.models.lora import DAPPLayer, DAPPPatchContainer
    fx = torch.load(os.path.join(golden_dir, "ref_lora_dapp_conv.pt"))
    st = fx["state"]

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.to_k = torch.nn.Linear(24, 32, bias=False)
            self.ff = torch.nn.Linear(32, 32, bias=True)
            self.proj = torch.nn.Conv2d(8, 16, 1)

    model = Net()
    model.load_state_dict({k.replace("._host", ""): v for k, v in st.items() if "._host." in k and k.split(".")[0] in ("to_k", "ff", "proj")})
    model = model.to(DEV).requires_grad_(False)
    for lname in ("to_k", "ff"):
        for lora_id, (branch, rank) in enumerate((("p", 4), ("n", 2))):
            DAPPLayer.wrap_layer(lora_id, getattr(model, lname), rank=rank, dropout=0.0, alpha=1.0, branch=branch, parent_block=model,
                                 host_name=lname)
    LoraLayer.wrap_layer(0, model.proj, rank=4, dropout=0.0, alpha=2.0, parent_block=model, host_name="proj")
    assert isinstance(model.to_k, DAPPPatchContainer) and type(model.to_k).__name__ == fx["container_types"]["to_k"]
    mine = model.state_dict()
    assert sorted(mine.keys()) == sorted(k for k in fx["state_keys_model"] if k.split(".")[0] in ("to_k", "ff", "proj"))
    with torch.no_grad():
        for k, v in mine.items():
            if "lora_block" in k:
                assert v.shape == st[k].shape, k
                v.copy_(st[k])
    xk = fx["xk"].to(DEV).requires_grad_(True)
    xf = fx["xf"].to(DEV).requires_grad_(True)
    xc = fx["xc"].to(DEV).requires_grad_(True)
    outs = {"to_k": model.to_k(xk), "ff": model.ff(xf), "proj": model.proj(xc)}
    for k, v in outs.items():
        assert v.shape == fx["outs"][k].shape and rel_l2(v, fx["outs"][k]) < 1e-2, k
    # the golden loss also contains the two 3x3 convolutions; their share of d(loss)/d(xc) is removed through the oracle
    sum((o ** 2).sum() for o in outs.values()).backward()
    assert rel_l2(xk.grad, fx["grad_in"]["xk"]) < 2e-2 and rel_l2(xf.grad, fx["grad_in"]["xf"]) < 2e-2
    for name, p in model.named_parameters():
        if "lora_block" in name:
            assert rel_l2(p.grad, fx["grads"][name]) < 3e-2, name


def test_tiny_unet_dapp_and_conv1x1_lora_forward_backward():
    """BASELINE config 5 topology at test size: DreamArtist++ pairs (type dapp, branch p rank 4 / branch n rank 2) on every
    Linear of the cross-attentions and feed-forwards, UNet batch = [negative half | positive half] (reference
    cfgs/train/examples/DreamArtist++.yaml, lora_layers_patch.py:102-133), plus a plain rank-4 LoRA on the 1x1 proj_in / proj_out
    convolutions (LoCon on 1x1 hosts).  noise_pred and every LoRA gradient against the fp32 oracle, whose DAPP / Conv2d semantics
    are pinned to the reference.  (The `layers` patterns name the PARENT modules: like in the reference, two config items that
    both match a leaf Linear by name re-wrap the stale leaf and orphan the first item's container -- cfg_net_tools.py:108-121.)"""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    pat = r".*\.attn2$|.*\.ff$"
    cfg = [{"type": "dapp", "branch": "p", "rank": 4, "alpha": 1.0, "dropout": 0.0, "layers": ["re:" + pat]},
           {"type": "dapp", "branch": "n", "rank": 2, "alpha": 1.0, "dropout": 0.0, "layers": ["re:" + pat]},
           {"rank": 4, "alpha": 2.0, "dropout": 0.0, "layers": [r"re:.*\.proj_in$", r"re:.*\.proj_out$"]}]
    _, group = make_hcpdiff(unet, None, cfg)
    lora = {}
    for idx, (branch, rank, alpha, patt, conv) in enumerate((("p", 4, 1.0, pat, False), ("n", 2, 1.0, pat, False),
                                                             (None, 4, 2.0, r".*\.proj_in$|.*\.proj_out$", True))):
        part = U.init_lora(spec, rank=rank, alpha=alpha, seed=11 + idx, up_std=0.05, pattern=patt, include_conv=conv, branch=branch)
        for layer, entries in part.items():
            lora.setdefault(layer, []).extend(entries)
    # copy the oracle factors into the product blocks: lora_block_<id> of a layer is the block of cfg item <id>
    named = dict(unet.named_modules())
    n_blocks = 0
    with torch.no_grad():
        for layer, entries in lora.items():
            cont = named[layer]
            for e in entries:
                bid = {"p": 0, "n": 1, None: 2}[e.branch]
                blk = getattr(cont, f"lora_block_{bid}")
                assert blk.layer.W_down.shape == e.W_down.shape and abs(float(blk.alpha) - e.alpha) < 1e-7, layer
                blk.layer.W_down.copy_(e.W_down)
                blk.layer.W_up.copy_(e.W_up)
                n_blocks += 1
    assert n_blocks == sum(1 for m in unet.modules() if isinstance(m, LoraLayer))
    lat, noise, t, ehs = U.synthetic_batch(4, spec)
    loss_ref, pred_ref, grads_ref = U.lora_step_loss_and_grads(sd, lora, lat, noise, t, ehs, spec)
    x_t = U.add_noise(lat, noise, t, U.ddpm_alphas_cumprod())
    pred = unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV)).sample
    assert rel_l2(pred, pred_ref) < 2e-2
    # the two halves must really have used different adapters: swapping the halves of the batch changes the result
    loss = F.mse_loss(pred, noise.to(DEV), reduction="none").mean()
    loss.backward()
    num = den = 0.0
    for layer, entries in lora.items():
        cont = named[layer]
        for e, (gd, gu) in zip(entries, grads_ref[layer]):
            blk = getattr(cont, f"lora_block_{ {'p': 0, 'n': 1, None: 2}[e.branch] }")
            for got, ref in ((blk.layer.W_down.grad, gd), (blk.layer.W_up.grad, gu)):
                num += float((got.cpu().double() - ref.double()).pow(2).sum())
                den += float(ref.double().pow(2).sum())
    assert math.sqrt(num / den) < 5e-2


@pytest.mark.parametrize("B,H,Cin,Cout,stride,ranks", [(2, 16, 64, 128, 1, (4,)), (2, 16, 128, 64, 2, (4, 8)), (1, 32, 64, 64, 1, (8,))])
def test_conv3x3_lora_fwd_bwd(B, H, Cin, Cout, stride, ranks):
    """Conv2d LoRA (LoCon) on a 3x3 convolution: y = conv(x, W + sum_b alpha_b W_up_b x W_down_b) (reference
    lora_layers_patch.py:91-98) through the factored kernels vs the materialised fp32 formula; x, W_down and W_up gradients."""
    from hcp_diffusion_b200.ops import ConvLoraRef
    x = rnd(B, H * H, Cin, seed=1).to(BF).requires_grad_(True)
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2)
    b = rnd(Cout, scale=0.1, seed=3)
    pack = ConvPack(w, b, stride)
    blocks = []
    for i, r in enumerate(ranks):
        down = rnd(r, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=10 + i).requires_grad_(True)
        up = rnd(Cout, r, 1, 1, scale=0.3, seed=20 + i).requires_grad_(True)
        blocks.append(ConvLoraRef(down, up, 0.25))
    pack.attach_lora(blocks)

    class G:
        pass
    g = G()
    g.pack = pack
    pack_lora([g])
    y = ops.conv3x3(pack, x, (B, H, H))
    xr = x.detach().float().view(B, H, H, Cin).permute(0, 3, 1, 2).requires_grad_(True)
    refs = [(blk.w_down.detach().clone().requires_grad_(True), blk.w_up.detach().clone().requires_grad_(True)) for blk in blocks]
    wp = bf(w)
    for d, u in refs:
        wp = wp + 0.25 * torch.einsum("or,rikl->oikl", u[:, :, 0, 0], d)
    yr = F.conv2d(xr, wp, b, stride=stride, padding=1)
    Ho = H // stride
    yr_nhwc = yr.permute(0, 2, 3, 1).reshape(B, Ho * Ho, Cout)
    assert rel_l2(y, yr_nhwc) < 1e-2
    dy = rnd(B, Ho * Ho, Cout, seed=6).to(BF)
    y.backward(dy)
    yr_nhwc.backward(dy.float())
    assert rel_l2(x.grad, xr.grad.permute(0, 2, 3, 1).reshape(B, H * H, Cin)) < 1e-2
    for blk, (d, u) in zip(blocks, refs):
        assert rel_l2(blk.w_down.grad, d.grad) < 2e-2
        assert rel_l2(blk.w_up.grad, u.grad) < 2e-2


def test_conv3x3_lora_container_standalone():
    """LoraLayer.wrap_layer on a 3x3 nn.Conv2d and a direct call of the container (NCHW in / out, like the reference layer)."""
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(64, 64, 3, padding=1).to(DEV).requires_grad_(False)
    holder = torch.nn.Module()
    holder.conv = conv
    blk = LoraLayer.wrap_layer(0, conv, rank=4, dropout=0.0, alpha=2.0, parent_block=holder, host_name="conv")
    with torch.no_grad():
        blk.layer.W_up.normal_(0, 0.2)
    x = rnd(2, 64, 16, 16, seed=3)
    y = holder.conv(x)
    wp = bf(conv.weight) + float(blk.alpha) * torch.einsum("or,rikl->oikl", blk.layer.W_up[:, :, 0, 0], blk.layer.W_down)
    yr = F.conv2d(bf(x), wp.detach(), conv.bias, padding=1)
    assert y.shape == yr.shape and rel_l2(y, yr) < 1e-2


def test_tiny_unet_locon_forward_backward():
    """BASELINE config 4's adapter placement at test size: LoRA rank 4 on every 3x3 / 1x1 convolution of the resnets and the
    down/up-samplers (reference cfgs/train/examples/locon.yaml pattern) -- noise_pred and all LoRA gradients vs the fp32 oracle."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels,
                                attention_head_dim=spec.num_heads, cross_attention_dim=spec.cross_attention_dim)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    pat = r".*\.resnets\.\d+\.conv[12]$|.*\.conv_shortcut$|.*samplers\.0\.conv$"
    _, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "dropout": 0.0, "layers": ["re:" + pat]}])
    lora = U.init_lora(spec, rank=4, alpha=1.0, seed=5, up_std=0.05, pattern=pat, include_conv=True)
    assert set(lora) == set(group.plugin_dict) and len(lora) > 40
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    loss_ref, pred_ref, grads_ref = U.lora_step_loss_and_grads(sd, lora, lat, noise, t, ehs, spec)
    x_t = U.add_noise(lat, noise, t, U.ddpm_alphas_cumprod())
    pred = unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV)).sample
    assert rel_l2(pred, pred_ref) < 2e-2
    F.mse_loss(pred, noise.to(DEV), reduction="none").mean().backward()
    num = den = 0.0
    for layer, blocks in grads_ref.items():
        blk = group[layer]
        for got, ref in ((blk.layer.W_down.grad, blocks[0][0]), (blk.layer.W_up.grad, blocks[0][1])):
            num += float((got.cpu().double() - ref.double()).pow(2).sum())
            den += float(ref.double().pow(2).sum())
    assert math.sqrt(num / den) < 5e-2


def unet_for_spec(spec):
    """Product UNet with the diffusers config keys of an oracle spec (SD1.x or SDXL topology)."""
    down = tuple("CrossAttnDownBlock2D" if a else "DownBlock2D" for a in spec.down_has_attn)
    up = tuple("CrossAttnUpBlock2D" if a else "UpBlock2D" for a in spec.up_has_attn)
    return UNet2DConditionModel(
        sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
        cross_attention_dim=spec.cross_attention_dim, down_block_types=down, up_block_types=up,
        transformer_layers_per_block=spec.transformer_depth, use_linear_projection=spec.use_linear_projection,
        addition_embed_type="text_time" if spec.addition_time_embed_dim else None, addition_time_embed_dim=spec.addition_time_embed_dim,
        projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)


@pytest.mark.parametrize("rank", [0, 4])
def test_tiny_sdxl_unet_forward_backward(rank):
    """SDXL topology (SURVEY 8f-4 / BASELINE config 4) at test size: no attention at the top level, transformer depth (2, 3),
    head dim 64, Linear proj_in/proj_out, `added_cond_kwargs` = {text_embeds, time_ids} (reference wrapper.py:57-75), LoRA on every
    attn / ff Linear (cfgs/train/examples/lora_sdxl.yaml) -- noise_pred and LoRA gradients against the fp32 oracle."""
    spec = U.TINY_XL
    sd = U.init_params(spec)
    unet = unet_for_spec(spec)
    unet.load_state_dict(sd)
    unet = unet.to(DEV).requires_grad_(False).eval()
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    added = U.synthetic_added_cond(2, spec)
    added_dev = {k: v.to(DEV) for k, v in added.items()}
    x_t = U.add_noise(lat, noise, t, U.ddpm_alphas_cumprod())
    if rank == 0:
        with torch.no_grad():
            pred_ref = U.unet_forward(sd, x_t, t, ehs, spec=spec, added_cond_kwargs=added)
            pred = unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV), added_cond_kwargs=added_dev).sample
        assert rel_l2(pred, pred_ref) < 2e-2
        with pytest.raises(ValueError):
            unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV))                 # the additional embedding is not optional
        return
    pat = r".*\.attn.?$|.*\.ff$"
    _, group = make_hcpdiff(unet, None, [{"rank": rank, "alpha": 1.0, "dropout": 0.0, "layers": ["re:" + pat]}])
    lora = U.init_lora(spec, rank=rank, seed=3, pattern=pat)
    assert set(lora) == set(group.plugin_dict)
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)
    loss_ref, pred_ref, grads_ref = U.lora_step_loss_and_grads(sd, lora, lat, noise, t, ehs, spec, added)
    pred = unet(x_t.to(DEV), t.to(DEV), ehs.to(DEV), added_cond_kwargs=added_dev).sample
    assert rel_l2(pred, pred_ref) < 2e-2
    F.mse_loss(pred, noise.to(DEV), reduction="none").mean().backward()
    num = den = 0.0
    for layer, blocks in grads_ref.items():
        blk = group[layer]
        for got, ref in ((blk.layer.W_down.grad, blocks[0][0]), (blk.layer.W_up.grad, blocks[0][1])):
            num += float((got.cpu().double() - ref.double()).pow(2).sum())
            den += float(ref.double().pow(2).sum())
    assert math.sqrt(num / den) < 5e-2


@pytest.mark.parametrize("use_graph", [False, True])
def test_cfg_denoising_loop_matches_oracle(use_graph):
    """Forward-only reuse (SURVEY 8f-4): the reference's CFG denoising loop (pipe_hook.py:115-150) with DDIM updates, 4 steps on the
    TINY UNet with a LoRA loaded, batch [negative | positive]; eager and captured-graph forwards against the oracle loop."""
    from hcp_diffusion_b200.sampling import CFGDenoiser
    spec = U.TINY
    sd = U.init_params(spec)
    unet, group, lora = build_product_unet(spec, sd, 4)
    g = torch.Generator().manual_seed(7)
    lat = torch.randn((2, 4, spec.sample_size, spec.sample_size), generator=g)
    pos = torch.randn((2, 77, spec.cross_attention_dim), generator=g)
    neg = torch.randn((2, 77, spec.cross_attention_dim), generator=g)
    ref = U.ddim_cfg_sample(sd, lat, pos, neg, 4, 5.0, spec=spec, lora=lora)
    out = CFGDenoiser(unet).sample(lat.to(DEV), pos.to(DEV), neg.to(DEV), num_inference_steps=4, guidance_scale=5.0, use_cuda_graph=use_graph)
    assert out.shape == ref.shape and rel_l2(out, ref) < 5e-2


def test_train_step_sdxl_added_cond_graph_matches_eager():
    """LoraTrainStep on the SDXL topology: `added_cond_kwargs` travel through the captured step (static device copies) -- the
    captured graph and the eager step produce the same losses and parameters."""
    spec = U.TINY_XL
    sd = U.init_params(spec)
    lat, noise, t, ehs = U.synthetic_batch(2, spec)
    added = U.synthetic_added_cond(2, spec)
    results = []
    for use_graph in (False, True):
        unet = unet_for_spec(spec)
        unet.load_state_dict(sd)
        unet = unet.to(DEV).requires_grad_(False).eval()
        groups, group = make_hcpdiff(unet, None, [{"rank": 4, "alpha": 1.0, "dropout": 0.0, "layers": [r"re:.*\.attn.?$", r"re:.*\.ff$"]}])
        lora = U.init_lora(spec, rank=4, seed=3, pattern=r".*\.attn.?$|.*\.ff$")
        with torch.no_grad():
            for layer, entries in lora.items():
                group[layer].layer.W_down.copy_(entries[0].W_down)
                group[layer].layer.W_up.copy_(entries[0].W_up)
        step = LoraTrainStep(unet, [p for g in groups for p in g["params"]], lr=1e-3, use_cuda_graph=use_graph)
        losses = [float(step.step(lat, noise, t, ehs, added).cpu()) for _ in range(4)]
        results.append((losses, step.flat.data.clone()))
    (l0, p0), (l1, p1) = results
    assert l0[-1] < l0[0]
    assert max(abs(a - b) for a, b in zip(l0, l1)) < 1e-3 * abs(l0[0]) and rel_l2(p1, p0) < 1e-3
