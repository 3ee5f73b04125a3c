"""Lion without a GPU: the restatement in tests/lion_ref.py against a hand-computed known answer, the engine's Lion state and
defaults, the entrypoint's option parsing and refusals, the schedulers' beta1 push, and the SD1.5 Lion fine-tuning config."""
import os

import pytest
import torch

from hcp_diffusion_b200 import train_ac
from hcp_diffusion_b200.engine import LoraTrainStep
from hcp_diffusion_b200.utils.config import load_config_with_cli

import lion_ref as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LION = "lion_pytorch.Lion"


def test_restatement_known_answer_three_steps():
    """lr 0.5, betas (0.5, 0.75); group A decays (wd 0.5: p x 0.75 every step), group B does not.  Every value is dyadic, so fp32
    holds each one exactly.  The case covers positive, negative and exactly-zero c (A[2] never has momentum; B[1] at step 3 has
    m b1 = -g (1 - b1)), and zero gradients that still move through the momentum (A[0], A[1] at step 2)."""
    a = torch.nn.Parameter(torch.ones(4))
    b = torch.nn.Parameter(torch.full((2,), 2.0))
    opt = L.Lion([{"params": [a], "weight_decay": 0.5}, {"params": [b]}], lr=0.5, betas=(0.5, 0.75))
    grads = [([1.0, -1.0, 0.0, 0.0], [0.0, 4.0]),
             ([0.0, 0.0, 0.0, 2.0], [0.0, -4.0]),
             ([-1.0, 0.0, 0.0, -1.0], [0.0, 0.25])]
    # hand-computed: p = 0.75 p - 0.5 sign(0.5 m + 0.5 g), m = 0.75 m + 0.25 g (A); the same without the 0.75 (B)
    want = [([0.25, 1.25, 0.75, 0.75], [0.25, -0.25, 0.0, 0.0], [2.0, 1.5], [0.0, 1.0]),
            ([-0.3125, 1.4375, 0.5625, 0.0625], [0.1875, -0.1875, 0.0, 0.5], [2.0, 2.0], [0.0, -0.25]),
            ([0.265625, 1.578125, 0.421875, 0.546875], [-0.109375, -0.140625, 0.0, 0.125], [2.0, 2.0], [0.0, -0.125])]
    for (ga, gb), (pa, ma, pb, mb) in zip(grads, want):
        a.grad, b.grad = torch.tensor(ga), torch.tensor(gb)
        opt.step()
        assert a.tolist() == pa and opt.state[a]["exp_avg"].tolist() == ma
        assert b.tolist() == pb and opt.state[b]["exp_avg"].tolist() == mb


def test_restatement_skips_parameters_without_gradient():
    p = torch.nn.Parameter(torch.ones(3))
    opt = L.Lion([p], lr=0.1, weight_decay=0.5)
    opt.step()
    assert p.tolist() == [1.0, 1.0, 1.0] and not opt.state[p]


def test_options_parsing_defaults_and_refusals():
    assert train_ac.optimizer_from_cfg({"_target_": LION, "_partial_": True}) == \
        ("lion", {"lr": 1e-4, "betas": (0.9, 0.99), "weight_decay": 0.0})
    name, opts = train_ac.optimizer_from_cfg({"_target_": LION, "lr": 3e-5, "betas": [0.95, 0.98], "weight_decay": 1e-2,
                                              "use_triton": True, "decoupled_weight_decay": False})
    assert name == "lion" and opts == {"lr": 3e-5, "betas": (0.95, 0.98), "weight_decay": 1e-2}
    with pytest.raises(TypeError, match="eps"):
        train_ac.optimizer_from_cfg({"_target_": LION, "eps": 1e-8})
    with pytest.raises(NotImplementedError, match="decoupled_weight_decay"):
        train_ac.optimizer_from_cfg({"_target_": LION, "decoupled_weight_decay": True})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "torch.optim.SGD"})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "somewhere.else.Lion"})


def cpu_step(optimizer, **kw):
    params = [torch.nn.Parameter(torch.zeros(5)), torch.nn.Parameter(torch.zeros(3, 2))]
    return LoraTrainStep(torch.nn.Identity(), [{"params": [params[0]], "lr": 1e-4}, {"params": [params[1]], "lr": 2e-4}],
                         optimizer=optimizer, **kw)


def test_engine_lion_state_and_defaults():
    lion = cpu_step("lion")
    assert lion.v is None and lion.m.numel() == lion.flat.numel == 8 + 8
    assert lion.optimizer_state_bytes == 4 * 16
    assert [b.data_ptr() for b in lion._opt_buffers()] == [lion.m.data_ptr()] + [s["step"].data_ptr() for s in lion.segments]
    assert lion.betas == (0.9, 0.99)
    for s, lr in zip(lion.segments, (1e-4, 2e-4)):
        assert s["hyper"].tolist() == pytest.approx([lr, 0.9, 0.99, 1e-8, 0.0])
    lion.set_hyper(1, lr=5e-5, beta1=0.85)
    assert lion.segments[1]["hyper"].tolist()[:2] == pytest.approx([5e-5, 0.85])
    adamw = cpu_step("adamw")                                   # AdamW's own defaults are unchanged
    assert adamw.betas == (0.9, 0.999) and adamw.optimizer_state_bytes == 2 * 4 * 16
    assert adamw.segments[0]["hyper"].tolist() == pytest.approx([1e-4, 0.9, 0.999, 1e-8, 1e-2])
    explicit = cpu_step("lion", betas=(0.95, 0.98), weight_decay=1e-2)
    assert explicit.segments[0]["hyper"].tolist() == pytest.approx([1e-4, 0.95, 0.98, 1e-8, 1e-2])
    with pytest.raises(ValueError, match="optimizer_kwargs"):
        cpu_step("lion", optimizer_kwargs={"weight_decay": 1e-2})
    with pytest.raises(ValueError, match="lion"):
        cpu_step("sgd")


def test_one_cycle_pushes_beta1_for_lion():
    class Fake:
        optimizer, betas = "lion", (0.9, 0.99)
        segments = [{"base_lr": 1e-3}, {"base_lr": 2e-3}]
        pushed = []

        def set_hyper(self, group, lr=None, beta1=None):
            self.pushed.append((group, lr, beta1))
    fake = Fake()
    step = train_ac.make_scheduler({"name": "one_cycle", "num_warmup_steps": 2, "num_training_steps": 10}, fake)
    assert fake.pushed[0][2] == pytest.approx(0.95)            # OneCycleLR starts at max_momentum and cycles beta1 down
    step()                                         # step 1 ends the warm-up phase (pct_start 0.2 of 10): max lr, base momentum
    assert fake.pushed[-2][2] == pytest.approx(0.85) and fake.pushed[-1][2] == pytest.approx(0.85)
    assert fake.pushed[-2][1] == pytest.approx(1e-3) and fake.pushed[-1][1] == pytest.approx(2e-3)


def test_ft_lion_yaml_loads():
    cfg = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "ft_lion_sd15_synthetic.yaml"))
    assert train_ac.optimizer_from_cfg(cfg.train.optimizer) == ("lion", {"lr": 1e-4, "betas": (0.9, 0.99), "weight_decay": 1e-2})
    assert list(cfg.unet[0].layers) == [""] and float(cfg.unet[0].lr) == 1e-6
    assert cfg.train.scheduler.name == "constant_with_warmup"
    assert (cfg.train.scheduler.num_warmup_steps, cfg.train.scheduler.num_training_steps) == (50, 600)
    assert cfg.tokenizer_pt.train is None and train_ac.images_per_step(cfg.data) == 4
