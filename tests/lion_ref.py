"""Restatement of lion_pytorch.Lion (the reference's cfgs/train/examples/Lion_optimizer.yaml optimizer) -- test infrastructure.

lion-pytorch's `Lion.step` / `update_fn` (Chen et al. 2023, "Symbolic Discovery of Optimization Algorithms", Program 1), per
parameter whose gradient exists, in this order:
    p = p * (1 - lr * wd);  c = m * beta1 + g * (1 - beta1);  p = p - lr * sign(c);  m = m * beta2 + g * (1 - beta2)
with the state `exp_avg` (m) zeros at the first step.  `reference_loop` puts it into oracle.step_ref.ReferenceLoop in place of
AdamW (clip_grad_norm_, accumulation, DDP averaging and EMA as there).
"""
from __future__ import annotations

import torch

from oracle import step_ref as S


class Lion(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-4, betas=(0.9, 0.99), weight_decay: float = 0.0):
        if lr <= 0.0:
            raise ValueError(f"lr {lr}")
        if not all(0.0 <= b <= 1.0 for b in betas):
            raise ValueError(f"betas {betas}")
        super().__init__(params, {"lr": lr, "betas": tuple(betas), "weight_decay": weight_decay})

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            lr, wd = group["lr"], group["weight_decay"]
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                if not state:
                    state["exp_avg"] = torch.zeros_like(p)
                m, g = state["exp_avg"], p.grad
                p.mul_(1.0 - lr * wd)
                c = m.mul(beta1).add(g, alpha=1.0 - beta1)
                p.add_(c.sign(), alpha=-lr)
                m.mul_(beta2).add_(g, alpha=1.0 - beta2)


def use_lion(ref: S.ReferenceLoop, betas=(0.9, 0.99), weight_decay: float = 0.0) -> S.ReferenceLoop:
    """Replace the reference loop's AdamW by Lion over the same parameter groups and learning rates."""
    ref.opt = Lion([{"params": g["params"], "lr": g["lr"]} for g in ref.opt.param_groups], lr=ref.opt.defaults["lr"], betas=betas,
                   weight_decay=weight_decay)
    return ref
