"""fp64 restatement of transformers.optimization.Adafactor.step (the reference's FT_sdxl.yaml optimizer) -- test infrastructure.

Pinned to the real class by tests/golden/ref_adafactor.pt (written by tests/golden/make_golden_adafactor.py) in
tests/test_adafactor.py.  `reference_loop` puts it into oracle.step_ref.ReferenceLoop in place of AdamW.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch

from oracle import step_ref as S

GOLDEN_SHAPES = [(5,), (1,), (3, 7), (77, 33), (64, 320), (8, 4, 3, 3), (6, 5, 1, 1), (2, 3, 4, 5)]
GOLDEN_STEPS = 6
GOLDEN_CASES: List[Dict] = [
    {"name": "defaults", "opts": {}},
    {"name": "manual_lr", "opts": {"lr": 1e-2, "relative_step": False}},
    {"name": "manual_lr_unscaled", "opts": {"lr": 1e-2, "relative_step": False, "scale_parameter": False}},
    {"name": "warmup_init", "opts": {"warmup_init": True}},
    {"name": "beta1", "opts": {"beta1": 0.9}},
    {"name": "weight_decay", "opts": {"lr": 1e-3, "relative_step": False, "weight_decay": 1e-3}},
    {"name": "clip_threshold", "opts": {}, "spike": 1000.0},
    {"name": "zero_init", "opts": {}, "zero_init": True},
]


def golden_inputs(case: Dict, seed: int = 0):
    """(initial parameters, gradients [step][tensor]) of one golden case, fp32.  The gradient grows by `spike` from step 4 on, so
    that rms(update) exceeds clip_threshold."""
    g = torch.Generator().manual_seed(seed)
    p0 = [torch.randn(s, generator=g) for s in GOLDEN_SHAPES]
    if case.get("zero_init"):
        p0 = [torch.zeros_like(p) for p in p0]
    grads = []
    for k in range(GOLDEN_STEPS):
        scale = case.get("spike", 1.0) if k >= 3 else 1.0
        grads.append([torch.randn(s, generator=g) * 0.1 * scale for s in GOLDEN_SHAPES])
    return p0, grads


def adafactor_step(p: torch.Tensor, grad: torch.Tensor, state: dict, lr=None, eps=(1e-30, 1e-3), clip_threshold=1.0, decay_rate=-0.8,
                   beta1=None, weight_decay=0.0, scale_parameter=True, relative_step=True, warmup_init=False) -> None:
    """One Adafactor step of tensor `p` (in place), in float64; `state` holds step, exp_avg_sq_row / _col or exp_avg_sq, exp_avg."""
    pd, gd = p.detach().double(), grad.detach().double()
    factored = pd.dim() >= 2
    if not state:
        state["step"] = 0
        if beta1 is not None:
            state["exp_avg"] = torch.zeros_like(gd)
        if factored:
            state["exp_avg_sq_row"] = torch.zeros(gd.shape[:-1], dtype=torch.float64)
            state["exp_avg_sq_col"] = torch.zeros(gd.shape[:-2] + gd.shape[-1:], dtype=torch.float64)
        else:
            state["exp_avg_sq"] = torch.zeros_like(gd)
    state["step"] += 1
    step = state["step"]
    rms_p = float(pd.norm() / math.sqrt(pd.numel()))
    lr_t = min(1e-6 * step if warmup_init else 1e-2, 1.0 / math.sqrt(step)) if relative_step else lr
    if scale_parameter:
        lr_t *= max(eps[1], rms_p)
    beta2t = 1.0 - math.pow(step, decay_rate)
    q = gd * gd + eps[0]
    if factored:
        row, col = state["exp_avg_sq_row"], state["exp_avg_sq_col"]
        row.mul_(beta2t).add_(q.mean(dim=-1), alpha=1.0 - beta2t)
        col.mul_(beta2t).add_(q.mean(dim=-2), alpha=1.0 - beta2t)
        u = (row / row.mean(dim=-1, keepdim=True)).rsqrt().unsqueeze(-1) * col.unsqueeze(-2).rsqrt() * gd
    else:
        v = state["exp_avg_sq"]
        v.mul_(beta2t).add_(q, alpha=1.0 - beta2t)
        u = v.rsqrt() * gd
    u = u / max(1.0, float(u.norm() / math.sqrt(u.numel())) / clip_threshold) * lr_t
    if beta1 is not None:
        m = state["exp_avg"]
        m.mul_(beta1).add_(u, alpha=1.0 - beta1)
        u = m
    pd = pd - weight_decay * lr_t * pd - u
    with torch.no_grad():
        p.copy_(pd.to(p.dtype))


class OracleAdafactor(torch.optim.Optimizer):
    """`adafactor_step` as a torch optimizer (per-group lr; the other options are optimizer-wide)."""

    def __init__(self, params, lr=None, **kw):
        super().__init__(params, {"lr": lr})
        self.kw = kw

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is not None:
                    adafactor_step(p, p.grad, self.state[p], lr=group["lr"], **self.kw)


def reference_loop(sd, lora, spec, optimizer_kwargs=None, **kw) -> S.ReferenceLoop:
    """oracle.step_ref.ReferenceLoop (clip, accumulation, EMA, CFG as there) with Adafactor instead of AdamW."""
    opts = dict(optimizer_kwargs or {})
    lr = opts.pop("lr", None)
    ref = S.ReferenceLoop(sd, lora, spec, lr=lr if lr is not None else 1e-4, **kw)
    groups = [{"params": g["params"], "lr": lr if "lrs" not in kw else g["lr"]} for g in ref.opt.param_groups]
    ref.opt = OracleAdafactor(groups, lr=lr, **opts)
    return ref
