"""Restatement of prodigyopt.Prodigy -- test infrastructure.

Written from the published `Prodigy.step` of prodigyopt 1.0 (Mishchenko & Defazio 2023, "Prodigy: An Expeditiously Adaptive
Parameter-Free Learner", Algorithm 3 with Adam).  prodigyopt is not installed where these tests run, so nothing pins this file to
the package: it is the algorithm as published, kept in the package's order of operations.  Per `step()`:

    lr = max over groups of lr_i (each lr_i equal to lr or 0, else RuntimeError);  beta3 = beta3 or sqrt(beta2)
    dlr = d lr (sqrt(1 - beta2^(k+1)) / (1 - beta1^(k+1)) with use_bias_correction);  D_num = beta3 D_num;  D_den = 0
    per parameter with a gradient: coupled decay g += wd p;  first call p0 = p, s = m = v = 0;  when lr_i > 0:
        D_num += (d / d0) dlr <g, p0 - p>;  m = beta1 m + d (1 - beta1) g;  v = beta2 v + d^2 (1 - beta2) g^2
        s = beta3 s + (d / d0) (d if safeguard_warmup else dlr) g;  D_den += sum |s|
    D_den == 0: return (nothing else changes)
    lr > 0: d_hat = d_coef D_num / D_den;  d = max(d, d_hat) if d == d0;  d_max = max(d_max, d_hat);  d = min(d_max, d growth_rate)
    per parameter: decoupled decay p -= wd dlr p;  p -= dlr m / (sqrt(v) + d eps)  (old dlr, new d);  k += 1

The scalars d, d_max, D_num (`d_numerator`) and k live in every param group, as in prodigyopt.  `use_prodigy` puts it into
oracle.step_ref.ReferenceLoop in place of AdamW (clip_grad_norm_, accumulation, DDP averaging and EMA as there).
"""
from __future__ import annotations

import math

import torch

from oracle import step_ref as S

LR_MESSAGE = "Setting different lr values in different parameter groups is only supported for values of 0"


class Prodigy(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1.0, betas=(0.9, 0.999), beta3=None, eps: float = 1e-8, weight_decay: float = 0.0,
                 decouple: bool = True, use_bias_correction: bool = False, safeguard_warmup: bool = False, d0: float = 1e-6,
                 d_coef: float = 1.0, growth_rate: float = float("inf")):
        if lr <= 0.0 or d0 <= 0.0:
            raise ValueError(f"lr {lr}, d0 {d0}")
        defaults = dict(lr=lr, betas=tuple(betas), beta3=beta3, eps=eps, weight_decay=weight_decay, d=d0, d0=d0, d_max=d0,
                        d_numerator=0.0, d_coef=d_coef, k=0, growth_rate=growth_rate, use_bias_correction=use_bias_correction,
                        decouple=decouple, safeguard_warmup=safeguard_warmup)
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        d_denom = 0.0
        group = self.param_groups[0]
        beta1, beta2 = group["betas"]
        beta3 = group["beta3"] if group["beta3"] is not None else math.sqrt(beta2)
        k = group["k"]
        d, d_max, d_coef = group["d"], group["d_max"], group["d_coef"]
        lr = max(g["lr"] for g in self.param_groups)
        bias_correction = (1 - beta2 ** (k + 1)) ** 0.5 / (1 - beta1 ** (k + 1)) if group["use_bias_correction"] else 1
        dlr = d * lr * bias_correction
        growth_rate, decouple = group["growth_rate"], group["decouple"]
        d_numerator = group["d_numerator"] * beta3
        for group in self.param_groups:
            decay, group_lr, d0 = group["weight_decay"], group["lr"], group["d0"]
            if group_lr not in [lr, 0.0]:
                raise RuntimeError(LR_MESSAGE)
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad
                if decay != 0 and not decouple:
                    grad.add_(p, alpha=decay)
                state = self.state[p]
                if "step" not in state:
                    state["step"] = 0
                    state["s"] = torch.zeros_like(p)
                    state["p0"] = p.detach().clone()
                    state["exp_avg"] = torch.zeros_like(p)
                    state["exp_avg_sq"] = torch.zeros_like(p)
                exp_avg, exp_avg_sq, s, p0 = state["exp_avg"], state["exp_avg_sq"], state["s"], state["p0"]
                if group_lr > 0.0:
                    d_numerator += (d / d0) * dlr * torch.dot(grad.flatten(), (p0 - p).flatten()).item()
                    exp_avg.mul_(beta1).add_(grad, alpha=d * (1 - beta1))
                    exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=d * d * (1 - beta2))
                    if group["safeguard_warmup"]:
                        s.mul_(beta3).add_(grad, alpha=(d / d0) * d)
                    else:
                        s.mul_(beta3).add_(grad, alpha=(d / d0) * dlr)
                    d_denom += s.abs().sum().item()
        if d_denom == 0:
            return None
        d_hat = d
        if lr > 0.0:
            d_hat = d_coef * d_numerator / d_denom
            if d == group["d0"]:
                d = max(d, d_hat)
            d_max = max(d_max, d_hat)
            d = min(d_max, d * growth_rate)
        for group in self.param_groups:
            group["d_numerator"] = d_numerator
            group["d_denom"] = d_denom
            group["d"], group["d_max"], group["d_hat"] = d, d_max, d_hat
            decay, eps = group["weight_decay"], group["eps"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                state["step"] += 1
                denom = state["exp_avg_sq"].sqrt().add_(d * eps)
                if decay != 0 and decouple:
                    p.add_(p, alpha=-decay * dlr)
                p.addcdiv_(state["exp_avg"], denom, value=-dlr)
            group["k"] = group["k"] + 1
        return None


def use_prodigy(ref: S.ReferenceLoop, **kw) -> S.ReferenceLoop:
    """Replace the reference loop's AdamW by Prodigy over the same parameter groups and learning rates."""
    ref.opt = Prodigy([{"params": g["params"], "lr": g["lr"]} for g in ref.opt.param_groups], lr=ref.opt.defaults["lr"], **kw)
    return ref
