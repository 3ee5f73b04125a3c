"""Prodigy without a GPU: the quirks of the restatement in tests/prodigy_ref.py, the engine's Prodigy state and defaults, the
entrypoint's option parsing and refusals, the lr rule in both, and the SD1.5 Prodigy LoRA config."""
import math
import os

import pytest
import torch

from hcp_diffusion_b200 import prodigy, train_ac
from hcp_diffusion_b200.engine import LoraTrainStep
from hcp_diffusion_b200.utils.config import load_config_with_cli

import prodigy_ref as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODIGY = "prodigyopt.Prodigy"


def params(seed=0, shapes=((6,), (3, 4))):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, generator=g, dtype=torch.float64)) for s in shapes]


def set_grads(ps, seed):
    g = torch.Generator().manual_seed(1000 + seed)
    for p in ps:
        p.grad = torch.randn(p.shape, generator=g, dtype=torch.float64)


def test_first_step_starts_from_d0():
    """p0 = p at the first call, so D_num = 0 and d_hat = 0: d stays d0, and the update is dlr m / (sqrt(v) + d eps) with
    m = d0 (1 - b1) g, v = d0^2 (1 - b2) g^2 and dlr = d0 lr."""
    ps = params()
    before = [p.detach().clone() for p in ps]
    opt = P.Prodigy(ps, lr=1.0, d0=1e-3)
    set_grads(ps, 0)
    grads = [p.grad.clone() for p in ps]
    opt.step()
    group = opt.param_groups[0]
    assert group["d"] == 1e-3 and group["d_max"] == 1e-3 and group["d_numerator"] == 0.0 and group["k"] == 1
    for p, b, g in zip(ps, before, grads):
        m, v = 1e-3 * 0.1 * g, 1e-6 * 0.001 * g * g
        torch.testing.assert_close(p.detach(), b - 1e-3 * m / (v.sqrt() + 1e-3 * 1e-8), rtol=1e-12, atol=0)
        assert torch.equal(opt.state[p]["p0"], b)


@pytest.mark.parametrize("growth_rate,bias_correction", [(float("inf"), False), (float("inf"), True), (1.02, False)])
def test_d_never_decreases_and_growth_rate_caps_it(growth_rate, bias_correction):
    """d is non-decreasing (d = min(d_max, d growth) with d_max a running max); a finite growth_rate caps each step's rise."""
    ps = params(1)
    opt = P.Prodigy(ps, lr=1.0, weight_decay=0.01, growth_rate=growth_rate, use_bias_correction=bias_correction)
    ds = [opt.param_groups[0]["d"]]
    for k in range(12):
        set_grads(ps, k % 3)                       # recurring gradients: the parameters travel, so D_num grows
        opt.step()
        ds.append(opt.param_groups[0]["d"])
    assert all(b >= a for a, b in zip(ds, ds[1:])), ds
    assert ds[-1] > ds[0]
    if math.isfinite(growth_rate):                 # the first move away from d0 (d = max(d, d_hat)) is not capped
        assert all(b <= a * growth_rate * (1 + 1e-15) for a, b in zip(ds, ds[1:]) if a != ds[0])
        assert sum(a != ds[0] and b == a * growth_rate for a, b in zip(ds, ds[1:])) >= 1


def test_all_zero_gradient_leaves_p_d_and_k():
    """D_den == 0 (every gradient zero at the first call): p, d, d_max, D_num and k stay; p0 is still captured."""
    ps = params(2)
    before = [p.detach().clone() for p in ps]
    opt = P.Prodigy(ps, lr=1.0, weight_decay=0.1)
    for p in ps:
        p.grad = torch.zeros_like(p)
    opt.step()
    g = opt.param_groups[0]
    assert (g["d"], g["d_max"], g["d_numerator"], g["k"]) == (1e-6, 1e-6, 0.0, 0)
    assert all(torch.equal(p.detach(), b) for p, b in zip(ps, before))
    assert all(torch.equal(opt.state[p]["p0"], b) for p, b in zip(ps, before))


def test_lr_zero_first_call_records_p0_and_skips():
    """The first step of constant_with_warmup runs at lr 0: no group feeds D_den, so the call is skipped, but p0 is recorded."""
    ps = params(3)
    opt = P.Prodigy(ps, lr=1.0)
    opt.param_groups[0]["lr"] = 0.0
    set_grads(ps, 0)
    before = [p.detach().clone() for p in ps]
    opt.step()
    assert opt.param_groups[0]["k"] == 0 and all(torch.equal(p.detach(), b) for p, b in zip(ps, before))
    assert all(torch.equal(opt.state[p]["p0"], b) for p, b in zip(ps, before))
    opt.param_groups[0]["lr"] = 1.0
    set_grads(ps, 1)
    opt.step()
    assert opt.param_groups[0]["k"] == 1 and not torch.equal(ps[0].detach(), before[0])


def test_lr_zero_group_only_decays():
    """A group at lr 0 keeps m = v = s = 0 and gets only the decoupled decay p (1 - wd dlr), with the global dlr."""
    live, frozen = params(4)
    opt = P.Prodigy([{"params": [live]}, {"params": [frozen], "lr": 0.0, "weight_decay": 0.25}], lr=1.0, d0=1e-2)
    for k in range(3):
        set_grads([live, frozen], k)
        f0 = frozen.detach().clone()
        dlr = opt.param_groups[0]["d"] * 1.0
        opt.step()
        torch.testing.assert_close(frozen.detach(), f0 - 0.25 * dlr * f0, rtol=1e-15, atol=0)
        st = opt.state[frozen]
        assert not st["exp_avg"].any() and not st["exp_avg_sq"].any() and not st["s"].any()


def test_coupled_decay_enters_the_gradient():
    """decouple=False adds wd p to the gradient before the moments (AdamW's L2 form); the decoupled step is then not applied."""
    a, b = params(5), params(5)
    oa = P.Prodigy(a, weight_decay=0.5, decouple=False)
    ob = P.Prodigy(b)
    for p, q in zip(a, b):
        p.grad = torch.ones_like(p)
        q.grad = torch.ones_like(q) + 0.5 * q.detach()
    oa.step()
    ob.step()
    for p, q in zip(a, b):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-15, atol=0)


def test_restatement_refuses_unequal_lrs():
    a, b = params(6)
    opt = P.Prodigy([{"params": [a]}, {"params": [b], "lr": 0.5}], lr=1.0)
    set_grads([a, b], 0)
    with pytest.raises(RuntimeError, match="only supported for values of 0"):
        opt.step()


def test_options_parsing_defaults_and_refusals():
    name, opts = train_ac.optimizer_from_cfg({"_target_": PRODIGY, "_partial_": True})
    assert name == "prodigy"
    assert opts == {"lr": 1.0, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.0, "beta3": None, "d0": 1e-6, "d_coef": 1.0,
                    "growth_rate": float("inf"), "use_bias_correction": False, "safeguard_warmup": False, "decouple": True}
    name, opts = train_ac.optimizer_from_cfg({"_target_": PRODIGY, "lr": 0.5, "betas": [0.95, 0.99], "beta3": 0.9, "eps": 1e-6,
                                              "weight_decay": 0.01, "decouple": False, "use_bias_correction": True,
                                              "safeguard_warmup": True, "d0": 1e-5, "d_coef": 0.5, "growth_rate": 1.05,
                                              "fsdp_in_use": False, "slice_p": 1})
    assert opts == {"lr": 0.5, "betas": (0.95, 0.99), "eps": 1e-6, "weight_decay": 0.01, "beta3": 0.9, "d0": 1e-5, "d_coef": 0.5,
                    "growth_rate": 1.05, "use_bias_correction": True, "safeguard_warmup": True, "decouple": False}
    with pytest.raises(TypeError, match="momentum"):
        train_ac.optimizer_from_cfg({"_target_": PRODIGY, "momentum": 0.9})
    with pytest.raises(NotImplementedError, match="fsdp_in_use"):
        train_ac.optimizer_from_cfg({"_target_": PRODIGY, "fsdp_in_use": True})
    with pytest.raises(NotImplementedError, match="slice_p"):
        train_ac.optimizer_from_cfg({"_target_": PRODIGY, "slice_p": 11})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "somewhere.else.Prodigy"})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "dadaptation.DAdaptAdam"})


def cpu_step(lrs=(1.0, 1.0), **kw):
    ps = [torch.nn.Parameter(torch.zeros(5)), torch.nn.Parameter(torch.zeros(3, 2))]
    return LoraTrainStep(torch.nn.Identity(), [{"params": [p], "lr": lr} for p, lr in zip(ps, lrs)], optimizer="prodigy", **kw)


def test_engine_prodigy_state_and_defaults():
    pd = cpu_step()
    assert pd.flat.numel == 16 and pd.optimizer_state_bytes == 16 * 16
    assert [b.data_ptr() for b in pd._opt_buffers()] == [b.data_ptr() for b in (pd.pd_p0, pd.pd_s, pd.m, pd.v, pd.pd_state, pd.pd_step)]
    assert pd.betas == (0.9, 0.999) and pd.eps == 1e-8
    assert pd.pd_hyper.tolist() == pytest.approx([0.9, 0.999, math.sqrt(0.999), 1e-8, 1e-6, 1.0, float("inf"), 4.0])
    assert pd.pd_state.tolist() == [1e-6, 1e-6, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    assert pd.pd_segs.view(torch.float64)[:, 2:].tolist() == [[1.0, 0.0], [1.0, 0.0]]
    assert pd.pd_segs[:, :2].tolist() == [[0, 8], [8, 8]] and pd.step_count is pd.pd_step
    assert pd.pd_work.numel() * 8 == prodigy.WORKSPACE_BYTES
    pd.set_lr(0.5)                                              # a scheduler scales every group together
    assert pd.pd_segs_f64[:, 2].tolist() == [0.5, 0.5] and float(pd.lr) == 0.5
    pd.set_hyper(1, lr=0.25, beta1=0.8)                          # only group 0's betas are Prodigy's
    pd.set_hyper(0, beta1=0.85)
    assert pd.pd_segs_f64[1, 2].item() == 0.25 and pd.pd_hyper[0].item() == 0.85
    opts = {"beta3": 0.9, "d0": 1e-4, "d_coef": 2.0, "growth_rate": 1.1, "use_bias_correction": True, "safeguard_warmup": True,
            "decouple": False}
    explicit = cpu_step(lrs=(0.0, 2.0), betas=(0.95, 0.99), eps=1e-6, weight_decay=0.01, optimizer_kwargs=opts)
    assert explicit.pd_hyper.tolist() == pytest.approx([0.95, 0.99, 0.9, 1e-6, 1e-4, 2.0, 1.1, 3.0])
    assert explicit.pd_state[0].item() == 1e-4 and explicit.pd_segs_f64[:, 3].tolist() == [0.01, 0.01]
    default_lr = LoraTrainStep(torch.nn.Identity(), [torch.nn.Parameter(torch.zeros(4))], optimizer="prodigy")
    assert default_lr.segments[0]["base_lr"] == 1.0
    with pytest.raises(ValueError, match="optimizer_kwargs"):
        cpu_step(optimizer_kwargs={"momentum": 0.9})
    with pytest.raises(ValueError, match="optimizer_kwargs"):   # the other optimizers' wording is unchanged
        LoraTrainStep(torch.nn.Identity(), [torch.nn.Parameter(torch.zeros(4))], optimizer="lion", optimizer_kwargs={"d0": 1e-6})
    with pytest.raises(ValueError, match="prodigy"):
        LoraTrainStep(torch.nn.Identity(), [torch.nn.Parameter(torch.zeros(4))], optimizer="dadapt")


def test_engine_refuses_unequal_lrs():
    with pytest.raises(RuntimeError, match="only supported for values of 0"):
        cpu_step(lrs=(1.0, 0.5))
    cpu_step(lrs=(0.0, 0.5))                                   # 0 and the largest lr are fine


def test_train_ac_items_with_unequal_lrs_are_refused():
    """What the entrypoint builds from two lora_unet items at lr 1.0 and 0.5 under prodigyopt.Prodigy is refused at construction."""
    from hcp_diffusion_b200.models import UNet2DConditionModel
    from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff
    name, opts = train_ac.optimizer_from_cfg({"_target_": PRODIGY})
    for lr2, refused in ((0.5, True), (1.0, False)):
        unet = UNet2DConditionModel(sample_size=8, block_out_channels=(32, 64, 64, 64), attention_head_dim=2, cross_attention_dim=32)
        unet.requires_grad_(False)
        items = [{"lr": 1.0, "rank": 2, "layers": [r"re:.*\.attn1$"]}, {"lr": lr2, "rank": 2, "layers": [r"re:.*\.attn2$"]}]
        groups, _ = make_hcpdiff(unet, None, items, default_lr=opts["lr"])
        build = lambda: LoraTrainStep(unet, groups, optimizer=name, betas=opts["betas"], eps=opts["eps"],  # noqa: E731
                                      weight_decay=opts["weight_decay"], optimizer_kwargs={k: opts[k] for k in prodigy.ENGINE_KEYS})
        if refused:
            with pytest.raises(RuntimeError, match="only supported for values of 0"):
                build()
        else:
            assert len(build().segments) == 2


def test_lora_prodigy_yaml_loads():
    cfg = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "lora_prodigy_sd15_synthetic.yaml"))
    name, opts = train_ac.optimizer_from_cfg(cfg.train.optimizer)
    assert name == "prodigy"
    assert opts["lr"] == 1.0 and opts["weight_decay"] == 0.01 and opts["use_bias_correction"] and opts["safeguard_warmup"]
    assert opts["decouple"] and opts["d0"] == 1e-6 and opts["growth_rate"] == float("inf")
    assert [float(it.lr) for it in cfg.lora_unet] == [1.0] and int(cfg.lora_unet[0].rank) == 8
    assert list(cfg.lora_unet[0].layers) == [r"re:.*\.attn.?$", r"re:.*\.ff$"]
    assert cfg.train.scheduler.name == "constant" and train_ac.images_per_step(cfg.data) == 4
