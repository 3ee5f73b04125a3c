"""`UNet2DConditionModel.gradient_checkpointing` (recompute regions over the BasicTransformerBlocks) and the time-embedding kernel at
batches beyond 16 rows (`pytest -m gpu` on an H100).

- The forward with the flag on is bit-identical to the flag off: the noise prediction of TINY and TINY_XL (LoRA with dropout on the
  attentions and the feed-forward, LoCon, DreamArtist++ containers, full fine-tuning).  The backward sums some gradients with fp32
  atomics (DESIGN §7), so the gradients agree to a rel-L2 of 2e-3 rather than bit for bit.
- The training-step tests of the other files run once with the flag off and once with it on (eager and under a CUDA graph: data
  groups with masks, accumulation 2, cfg_scale, text-encoder LoRA, the SDXL pair, full fine-tuning).  The flag-on runs are those
  tests' own comparisons with the reference loop, so the same tolerances apply; the two runs' first losses agree to 1e-5 relative
  and all their losses to 2e-3.
- The attention forward kernel is launched as often with the flag on as off, and a region saves for its backward exactly its input,
  the cross-attention context, both attention outputs and both LSE tensors.
- hcp_skinny_linear at M = 1 / 16 / 17 / 40 / 100 rows against float64, rows of a large-M call equal to the same rows in 16-row calls,
  and TINY LoRA steps at batch 17 and 40 beside the reference loop.
"""
import math

import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

import test_gpu_data_groups as DG  # noqa: E402
import test_gpu_fullft as FT  # noqa: E402
import test_gpu_more as MO  # noqa: E402
import test_gpu_norm_wgrad_edges as E  # noqa: E402
import test_gpu_sdxl_te as XL  # noqa: E402
import test_gpu_step as ST  # noqa: E402
import test_gpu_te_step as TE  # noqa: E402

from hcp_diffusion_b200 import ops  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.models.lora import DAPPLayer  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture
def checkpointing(monkeypatch):
    """Every UNet2DConditionModel built while this is active has gradient checkpointing on; returns a switch for it."""
    state = {"on": False}
    init = UNet2DConditionModel.__init__

    def patched(self, *args, **kwargs):
        init(self, *args, **kwargs)
        if state["on"]:
            self.enable_gradient_checkpointing()
    monkeypatch.setattr(UNet2DConditionModel, "__init__", patched)
    return state


@pytest.fixture
def losses(monkeypatch):
    """Records a copy of every loss LoraTrainStep.step / step_groups returns."""
    got = []
    for name in ("step", "step_groups"):
        orig = getattr(LoraTrainStep, name)

        def wrapped(self, *args, _orig=orig, **kwargs):
            out = _orig(self, *args, **kwargs)
            got.append(out.detach().clone())
            return out
        monkeypatch.setattr(LoraTrainStep, name, wrapped)
    return got


# ----------------------------------------------------------------------------------------------------------------------
# the training-step tests of the other files, flag off then on: the reference-loop checks pass with it on, the losses agree
# ----------------------------------------------------------------------------------------------------------------------
STEP_CASES = {
    "lora_eager": (ST.test_tiny_train_step_matches_reference_loop, (False,)),
    "lora_graph": (ST.test_tiny_train_step_matches_reference_loop, (True,)),
    "accum2_two_groups_minsnr_ema": (ST.test_tiny_train_step_accumulation_two_groups_minsnr_ema, ()),
    "cfg_scale": (ST.test_tiny_dreamartist_cfg_step_matches_reference_loop, ()),
    "groups_masks_eager": (DG.test_tiny_lora_groups_match_reference_loop, (False, 1)),
    "groups_masks_graph_accum2": (DG.test_tiny_lora_groups_match_reference_loop, (True, 2)),
    "full_ft": (FT.test_tiny_full_finetune_steps_match_reference_loop, ()),
    "te_lora_eager": (TE.test_joint_te_unet_steps_match_reference_loop, (False, 1.0)),
    "te_lora_graph": (TE.test_joint_te_unet_steps_match_reference_loop, (True, 1.0)),
    "sdxl_pair_graph": (XL.test_joint_sdxl_te_unet_steps_match_reference_loop, ("adamw", 1, False, True)),
    "sdxl_pair_eager": (XL.test_joint_sdxl_te_unet_steps_match_reference_loop, ("adamw", 0, True, False)),
}


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_training_steps_match_reference_loop_with_the_flag_on(case, checkpointing, losses):
    fn, args = STEP_CASES[case]
    runs = []
    for on in (False, True):
        checkpointing["on"] = on
        losses.clear()
        ops.set_dropout_seed(1234)
        fn(*args)
        runs.append(torch.cat([x.flatten() for x in losses]).cpu())
    assert runs[0].numel() >= 3
    assert abs(float(runs[1][0]) / float(runs[0][0]) - 1) < 1e-5, (runs[0], runs[1])          # the first loss: the forward alone
    assert rel(runs[1], runs[0]) < 2e-3, (runs[0], runs[1])


def test_dropout_and_locon_tests_pass_with_the_flag_on(checkpointing):
    checkpointing["on"] = True
    MO.test_tiny_unet_trains_with_dropout_under_cuda_graph()
    MO.test_tiny_unet_shipped_locon_yaml_items_match_oracle()


# ----------------------------------------------------------------------------------------------------------------------
# one forward / backward of the UNet: the prediction bit for bit, the gradients, attention launches, saved tensors
# ----------------------------------------------------------------------------------------------------------------------
def _init_up(group, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    with torch.no_grad():
        for blk in group.plugin_dict.values():
            blk.layer.W_up.copy_(torch.randn(blk.layer.W_up.shape, generator=g, device=DEV) * 0.05)


def setup_lora_dropout(unet):
    _, group = make_hcpdiff(unet, None, [{"lr": 1e-3, "rank": 4, "dropout": 0.1, "layers": [r"re:.*\.attn.?$", r"re:.*\.ff$"]}])
    _init_up(group, 1)


def setup_locon(unet):
    _, group = make_hcpdiff(unet, None, [{"lr": 1e-3, "rank": 8, "layers": [r"re:.*\.attn.?$", r"re:.*\.resnets$", r"re:.*\.proj_in$"]}])
    _init_up(group, 2)


def setup_dapp(unet):
    torch.manual_seed(3)
    for m in unet.modules():
        if type(m).__name__ == "Attention":
            for lname in ("to_q", "to_k", "to_v"):
                for lora_id, (branch, rank) in enumerate((("p", 4), ("n", 2))):
                    blk = DAPPLayer.wrap_layer(lora_id, getattr(m, lname), rank=rank, dropout=0.0, alpha=1.0, branch=branch, parent_block=m,
                                               host_name=lname)
                    with torch.no_grad():
                        nn.init.normal_(blk.layer.W_up, std=0.05)
    unet.to(DEV)


def setup_full(unet):
    make_hcpdiff(unet, [{"lr": 1e-5, "layers": [""]}], None)


SETUPS = {"lora_dropout": setup_lora_dropout, "locon": setup_locon, "dapp": setup_dapp, "full": setup_full}


def one_pass(spec, setup, on, B=4, ehs_grad=False, saved=None):
    """(pred, gradients, attention-forward launches) of one forward / backward of a freshly built UNet."""
    torch.manual_seed(0)                         # the adapters' initial factors
    unet = DG.tiny_unet(U.init_params(spec), spec)
    setup(unet)
    if on:
        unet.enable_gradient_checkpointing()
    lat, noise, t, ehs = U.synthetic_batch(B, spec, seed=11)
    kw = {}
    if spec.addition_time_embed_dim:
        kw["added_cond_kwargs"] = {k: v.to(DEV) for k, v in U.synthetic_added_cond(B, spec, seed=12).items()}
    ehs = ehs.to(DEV).requires_grad_(ehs_grad)
    ops.set_dropout_seed(99)
    ops._Drop.site = 0                           # the pass starts at the first dropout call site, as a training step does
    n_attn = [0]
    real_call = ops.call

    def counting(name, *args):
        if name.startswith("hcp_attn_fwd"):
            n_attn[0] += 1
        return real_call(name, *args)
    ops.call = counting
    try:
        if saved is not None:
            with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(t) or t, lambda t: t):
                pred = unet(lat.to(DEV), t.to(DEV), ehs, **kw).sample
        else:
            pred = unet(lat.to(DEV), t.to(DEV), ehs, **kw).sample
        g = torch.randn(pred.shape, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV)
        pred.backward(g)
    finally:
        ops.call = real_call
    params = [p for p in unet.parameters() if p.requires_grad]
    grads = [None if p.grad is None else p.grad.clone() for p in params] + ([ehs.grad.clone()] if ehs_grad else [])
    return pred.detach(), grads, n_attn[0]


@pytest.mark.parametrize("spec_name", ["TINY", "TINY_XL"])
@pytest.mark.parametrize("mode", list(SETUPS))
def test_forward_bit_identical_and_gradients_match(spec_name, mode):
    spec = getattr(U, spec_name)
    ehs_grad = mode == "lora_dropout"            # the text-embedding gradient through the per-attention aliases
    off = one_pass(spec, SETUPS[mode], False, ehs_grad=ehs_grad)
    on = one_pass(spec, SETUPS[mode], True, ehs_grad=ehs_grad)
    assert torch.equal(off[0], on[0])
    assert len(off[1]) == len(on[1]) > 0
    assert sum(g is not None for g in off[1]) > 0
    for a, b in zip(off[1], on[1]):
        assert (a is None and b is None) or rel(b, a) < 2e-3
    assert off[2] == on[2] > 0                   # the attention forward is never launched again by the recompute


def test_region_saves_input_context_outputs_and_lse_only():
    """Every tensor a region keeps for the backward passes through saved_tensors_hooks: per block exactly its input, the context,
    o1, lse1, o2 and lse2, and the whole pass keeps fewer bytes than with the flag off."""
    spec = U.TINY
    unet = DG.tiny_unet(U.init_params(spec), spec)
    n_blocks = sum(1 for m in unet.modules() if type(m).__name__ == "BasicTransformerBlock")
    nbytes = lambda ts: sum(t.numel() * t.element_size() for t in ts)   # noqa: E731
    saved_off, saved_on = [], []
    one_pass(spec, setup_lora_dropout, False, B=2, saved=saved_off)
    region_saved = []
    real = ops.CheckpointFn.forward

    def spy(ctx, run, n_in, *args):
        out = real(ctx, run, n_in, *args)
        region_saved.append([t for t in ctx.to_save if t is not None])
        return out
    ops.CheckpointFn.forward = staticmethod(spy)
    try:
        one_pass(spec, setup_lora_dropout, True, B=2, saved=saved_on)
    finally:
        ops.CheckpointFn.forward = staticmethod(real)
    print({"saved_off_MB": nbytes(saved_off) / 2 ** 20, "saved_on_MB": nbytes(saved_on) / 2 ** 20})
    assert nbytes(saved_on) < nbytes(saved_off)
    assert len(region_saved) == n_blocks
    hooked = {id(t) for t in saved_on}
    for ts in region_saved:
        assert len(ts) == 6 and all(id(t) in hooked for t in ts)
        h, ctx_t, o1, l1, o2, l2 = ts
        assert o1.shape == o2.shape == h.shape and o1.dtype == o2.dtype == h.dtype == torch.bfloat16
        assert l1.dtype == l2.dtype == torch.float32 and l1.shape[0] == h.shape[0] and l1.shape[2] == h.shape[1] and l1.shape == l2.shape
        assert ctx_t.shape[:2] == (2, 77)


def test_sd15_config2_peak_memory_is_lower():
    peaks = []
    for on in (False, True):
        unet = DG.tiny_unet(U.init_params(U.SD15), U.SD15)
        groups, _ = make_hcpdiff(unet, None, [{"rank": 8, "alpha": 1.0, "dropout": 0.0, "lr": 1e-4, "layers": [r"re:.*\.attn.?$"]}])
        if on:
            unet.enable_gradient_checkpointing()
        step = LoraTrainStep(unet, groups, lr=1e-4, use_cuda_graph=False)
        lat, noise, t, ehs = U.synthetic_batch(4, U.SD15, seed=1)
        step.step(lat, noise, t, ehs)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step.step(lat, noise, t, ehs)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del step, unet, groups
        torch.cuda.empty_cache()
    print({"peak_off_MB": peaks[0] / 2 ** 20, "peak_on_MB": peaks[1] / 2 ** 20})
    assert peaks[1] < 0.75 * peaks[0]


# ----------------------------------------------------------------------------------------------------------------------
# the time-embedding kernel beyond 16 rows
# ----------------------------------------------------------------------------------------------------------------------
def skinny(x, w, b, M, K, N, in_mode, out_silu):
    buf, y = E.flat_f32(M * N)
    call("hcp_skinny_linear", x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, in_mode, out_silu, y.data_ptr(), stream_ptr())
    E.flat_check("skinny y", buf, M * N)
    return y.view(M, N)


@pytest.mark.parametrize("M", [1, 16, 17, 40, 100])
@pytest.mark.parametrize("K,N,in_mode,out_silu", [(320, 1283, 2, 1), (1280, 1283, 1, 0), (2816, 1280, 0, 1), (514, 13, 0, 0)])
def test_skinny_linear_any_rows_matches_fp64_and_16_row_calls(M, K, N, in_mode, out_silu):
    x = (torch.arange(M, dtype=torch.float32, device=DEV) * 37.0 % 1000.0) if in_mode == 2 else E.rnd(M, K, seed=1, dtype=torch.float32)
    w = E.rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    b = E.rnd(N, scale=0.3, seed=3, dtype=torch.float32)
    y = skinny(x, w, b, M, K, N, in_mode, out_silu)
    xi = E.sinusoid64(x, K) if in_mode == 2 else x.double()
    if in_mode == 1:
        xi = torch.nn.functional.silu(xi)
    ref = xi @ w.double().t() + b.double()
    if out_silu:
        ref = torch.nn.functional.silu(ref)
    E.compare(f"skinny M{M} K{K} N{N}", y, ref, E.F32SUM if in_mode != 2 else E.F32SIN, block=(M, 8))
    for m0 in range(0, M, 16):                   # the same rows launched 16 at a time: the same bits
        m1 = min(M, m0 + 16)
        part = skinny(x[m0:m1].contiguous(), w, b, m1 - m0, K, N, in_mode, out_silu)
        assert torch.equal(part, y[m0:m1])


@pytest.mark.parametrize("batch", [17, 40])
def test_tiny_lora_steps_beyond_16_images_match_reference_loop(batch):
    ST.check(ST.run_side_by_side(U.TINY, batch=batch, rank=4, steps=3, lr=1e-3, use_graph=True))


def test_step_groups_beyond_16_images_match_reference_loop(monkeypatch):
    """Data groups of 12 masked + 9 images (21 per pass) with the checks of the data-group test."""
    real = DG.group_batches
    monkeypatch.setattr(DG, "group_batches", lambda spec, sizes, it, **kw: real(spec, [12, 9], it, **kw))
    DG.test_tiny_lora_groups_match_reference_loop(True, 1)
