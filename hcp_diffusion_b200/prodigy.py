"""Prodigy over the flat parameter buffer: option parsing and the device tables of `hcp_prodigy_flat`.

The optimizer is `prodigyopt.Prodigy` (Mishchenko & Defazio, "Prodigy: An Expeditiously Adaptive Parameter-Free Learner", 2023):
Adam's update scaled by a step size d that the optimizer estimates from sum g (p0 - p) over sum |s| across every trainable
parameter.  The kernel (csrc/optim.cu) keeps d and its companions in an fp64 block on the device, so the estimate never leaves the
GPU.  Per parameter it keeps p0 (the parameters at the first call), s, m and v: 16 B of fp32 state.

  segments  hcp_prodigy_segment [groups]: {offset, count, lr, weight_decay}, lr and weight_decay fp64
  hyper     fp64 [8]: {beta1, beta2, beta3, eps, d0, d_coef, growth_rate, flags}
  state     fp64 [8]: {d, d_max, D_num, k, initialised, skipped, dlr, unused}
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

# prodigyopt.Prodigy.__init__ keywords and defaults (slice_p arrived in prodigyopt 1.1; its default keeps the 1.0 algorithm)
DEFAULTS = {"lr": 1.0, "betas": (0.9, 0.999), "beta3": None, "eps": 1e-8, "weight_decay": 0.0, "decouple": True,
            "use_bias_correction": False, "safeguard_warmup": False, "d0": 1e-6, "d_coef": 1.0, "growth_rate": float("inf"),
            "fsdp_in_use": False, "slice_p": 1}
# the keys LoraTrainStep takes in optimizer_kwargs (lr / betas / eps / weight_decay are its own arguments)
ENGINE_KEYS = ("beta3", "d0", "d_coef", "growth_rate", "use_bias_correction", "safeguard_warmup", "decouple")
LR_MESSAGE = "Setting different lr values in different parameter groups is only supported for values of 0"
FLAG_BIAS_CORRECTION, FLAG_SAFEGUARD_WARMUP, FLAG_DECOUPLE = 1, 2, 4
HYPER, STATE, WORKSPACE_BYTES = 8, 8, 16384        # HCP_PRODIGY_* of include/hcp_b200.h

SEGMENT_DTYPE = np.dtype([("offset", "<i8"), ("count", "<i8"), ("lr", "<f8"), ("weight_decay", "<f8")])


def check_options(kw: Optional[dict]) -> dict:
    """The constructor keys of prodigyopt.Prodigy with its defaults.  An unknown key is a TypeError (as the constructor raises);
    `fsdp_in_use: True` and `slice_p` other than 1 are refused with NotImplementedError."""
    kw = dict(kw or {})
    unknown = sorted(set(kw) - set(DEFAULTS))
    if unknown:
        raise TypeError(f"Prodigy.__init__() got unexpected keyword arguments {unknown}")
    out = {**DEFAULTS, **kw}
    if out["fsdp_in_use"]:
        raise NotImplementedError("prodigyopt.Prodigy with fsdp_in_use: True is not supported (the engine is data-parallel, not FSDP)")
    if int(out["slice_p"]) != 1:
        raise NotImplementedError(f"prodigyopt.Prodigy with slice_p={out['slice_p']!r} is not supported (only 1)")
    betas = tuple(float(b) for b in out["betas"])
    if len(betas) != 2:
        raise ValueError(f"Prodigy betas {out['betas']!r}: two values (beta1, beta2)")
    opts = {"lr": float(out["lr"]), "betas": betas, "eps": float(out["eps"]), "weight_decay": float(out["weight_decay"])}
    return {**opts, **engine_options({k: out[k] for k in ENGINE_KEYS})}


def engine_options(kw: Optional[dict]) -> dict:
    """LoraTrainStep's `optimizer_kwargs` for Prodigy: the keys of ENGINE_KEYS with prodigyopt's defaults."""
    kw = dict(kw or {})
    unknown = sorted(set(kw) - set(ENGINE_KEYS))
    if unknown:
        raise ValueError(f"optimizer_kwargs for Prodigy take {list(ENGINE_KEYS)} (lr / betas / eps / weight_decay are arguments of "
                         f"their own); unknown: {unknown}")
    out = {**{k: DEFAULTS[k] for k in ENGINE_KEYS}, **kw}
    beta3 = out["beta3"]
    d0 = float(out["d0"])
    if d0 <= 0.0:
        raise ValueError(f"Prodigy d0 {d0!r} must be positive")
    return {"beta3": None if beta3 is None else float(beta3), "d0": d0, "d_coef": float(out["d_coef"]),
            "growth_rate": float(out["growth_rate"]), "use_bias_correction": bool(out["use_bias_correction"]),
            "safeguard_warmup": bool(out["safeguard_warmup"]), "decouple": bool(out["decouple"])}


def check_lrs(lrs) -> None:
    """prodigyopt's rule: every group's lr is the largest one or 0 (it raises RuntimeError in step(); here at construction)."""
    top = max(lrs) if lrs else 0.0
    if any(lr not in (top, 0.0) for lr in lrs):
        raise RuntimeError(LR_MESSAGE)


def hyper_row(opts: dict, beta1: float, beta2: float, eps: float) -> list:
    """The fp64 hyper block: beta3 defaults to sqrt(beta2), as in prodigyopt."""
    beta3 = math.sqrt(beta2) if opts["beta3"] is None else opts["beta3"]
    flags = (FLAG_BIAS_CORRECTION * opts["use_bias_correction"] + FLAG_SAFEGUARD_WARMUP * opts["safeguard_warmup"]
             + FLAG_DECOUPLE * opts["decouple"])
    return [beta1, beta2, beta3, eps, opts["d0"], opts["d_coef"], opts["growth_rate"], float(flags)]


def initial_state(d0: float) -> list:
    return [d0, d0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]


def segment_table(segments) -> np.ndarray:
    """[(offset, count, lr, weight_decay)] -> the packed hcp_prodigy_segment table."""
    tab = np.zeros(len(segments), dtype=SEGMENT_DTYPE)
    for i, (off, cnt, lr, wd) in enumerate(segments):
        tab[i] = (off, cnt, lr, wd)
    return tab
