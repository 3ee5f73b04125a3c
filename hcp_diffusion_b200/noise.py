"""`model.noise_scheduler` (reference cfgs/train/train_base.yaml:76, read at hcpdiff/train_ac.py:211-214) resolved into what the
training step computes with: the `alphas_cumprod` table of length T = `num_train_timesteps` (add_noise and the Min-SNR weights,
hcpdiff/loss/min_snr_loss.py:14-19) and, for `PyramidNoiseScheduler`, its pyramid parameters.

Accepted `_target_`s, by name as `train_ac.optimizer_from_cfg` takes optimizers:
  * `diffusers.DDPMScheduler` with its constructor keys.  Only `num_train_timesteps`, `beta_start`, `beta_end`, `beta_schedule`
    ('linear', 'scaled_linear', 'squaredcos_cap_v2') and `rescale_betas_zero_snr` touch the forward process; the others
    (`prediction_type`, `clip_sample`, ...) only steer sampling and are accepted unread.  `trained_betas` is refused.
  * `diffusers.DDPMScheduler.from_pretrained` (`pretrained_model_name_or_path`, `subfolder`): reads the local
    `<path>/<subfolder>/scheduler_config.json` diffusers would read; keys outside the forward process are ignored, as diffusers
    ignores them, and constructor keys given next to the path override the file's.
  * `hcpdiff.noise.ZeroTerminalScheduler(base_scheduler)` (hcpdiff/noise/zero_terminal.py): the base's betas rescaled to zero
    terminal SNR (arXiv 2305.08891, Algorithm 1) in float32, so alphas_cumprod[T-1] == 0.
  * `hcpdiff.noise.PyramidNoiseScheduler(base_scheduler, level=10, discount=0.9, step_size=2., resize_mode='bilinear')`
    (hcpdiff/noise/pyramid_noise.py), outermost.

`ZeroTerminalScheduler` around a `PyramidNoiseScheduler` is refused: the reference's NoiseBase.__setattr__ then stores the rescaled
tables on the pyramid wrapper instead of on the DDPMScheduler whose add_noise runs, so its x_t keeps the original table while the
loss reads the rescaled one.  `PyramidNoiseScheduler(ZeroTerminalScheduler(...))` rescales both.
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
from typing import Optional

import torch

from ._lib import PYRAMID_MAX_LEVEL

DDPM_DEFAULTS = {"num_train_timesteps": 1000, "beta_start": 0.0001, "beta_end": 0.02, "beta_schedule": "linear", "trained_betas": None,
                 "rescale_betas_zero_snr": False}
# DDPMScheduler.__init__ keys (diffusers <= 0.26.1) that do not change the forward process or the training loss
DDPM_SAMPLING_KEYS = {"variance_type", "clip_sample", "prediction_type", "thresholding", "dynamic_thresholding_ratio", "clip_sample_range",
                      "sample_max_value", "timestep_spacing", "steps_offset"}
PYRAMID_DEFAULTS = {"level": 10, "discount": 0.9, "step_size": 2.0, "resize_mode": "bilinear"}


@dataclasses.dataclass
class NoiseSchedule:
    """alphas_cumprod fp32 [T] (CPU); pyramid None or {'level', 'discount', 'step_size'}."""
    alphas_cumprod: torch.Tensor
    pyramid: Optional[dict] = None

    @property
    def num_train_timesteps(self) -> int:
        return int(self.alphas_cumprod.numel())

    @property
    def zero_terminal(self) -> bool:
        return float(self.alphas_cumprod[-1]) == 0.0


def ddpm_betas(num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
               beta_schedule: str = "linear") -> torch.Tensor:
    """DDPMScheduler.__init__'s betas, in diffusers' float32 arithmetic."""
    T = int(num_train_timesteps)
    if T < 2:
        raise ValueError(f"num_train_timesteps={T}: at least 2")
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, T, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, T, dtype=torch.float32) ** 2
    if beta_schedule == "squaredcos_cap_v2":                # betas_for_alpha_bar, cosine alpha_bar, max_beta 0.999
        def alpha_bar(t):
            return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
        return torch.tensor([min(1 - alpha_bar((i + 1) / T) / alpha_bar(i / T), 0.999) for i in range(T)], dtype=torch.float32)
    raise NotImplementedError(f"DDPMScheduler beta_schedule={beta_schedule!r}: one of 'linear', 'scaled_linear', 'squaredcos_cap_v2'")


def rescale_zero_terminal_snr(betas: torch.Tensor) -> torch.Tensor:
    """ZeroTerminalScheduler.rescale_zero_terminal_snr (zero_terminal.py:13-42), float32."""
    alphas_bar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
    a0, aT = alphas_bar_sqrt[0].clone(), alphas_bar_sqrt[-1].clone()
    alphas_bar_sqrt -= aT
    alphas_bar_sqrt *= a0 / (a0 - aT)
    alphas_bar = alphas_bar_sqrt ** 2
    alphas = torch.cat([alphas_bar[0:1], alphas_bar[1:] / alphas_bar[:-1]])
    return 1 - alphas


def _kwargs(node) -> dict:
    return {k: v for k, v in dict(node).items() if k not in ("_target_", "_partial_")}


def _ddpm(kw: dict, where: str) -> torch.Tensor:
    if kw.get("trained_betas") is not None:
        raise NotImplementedError(f"{where}: trained_betas is not supported; give beta_start / beta_end / beta_schedule")
    opts = {**DDPM_DEFAULTS, **{k: v for k, v in kw.items() if k in DDPM_DEFAULTS}}
    betas = ddpm_betas(opts["num_train_timesteps"], float(opts["beta_start"]), float(opts["beta_end"]), str(opts["beta_schedule"]))
    return rescale_zero_terminal_snr(betas) if opts["rescale_betas_zero_snr"] else betas


def _resolve(node, inside_zero_terminal: bool = False):
    """-> (betas fp32 [T], pyramid options or None)."""
    if not isinstance(node, dict) and not hasattr(node, "items"):
        raise TypeError(f"model.noise_scheduler: expected a mapping with _target_, got {type(node).__name__}")
    target = str(node.get("_target_", ""))
    name = target.rsplit(".", 1)[-1]
    kw = _kwargs(node)
    if target.startswith("diffusers.") and target.endswith("DDPMScheduler.from_pretrained"):
        path, sub = kw.pop("pretrained_model_name_or_path", None), kw.pop("subfolder", None) or ""
        if path is None:
            raise ValueError("DDPMScheduler.from_pretrained: pretrained_model_name_or_path is required")
        cfg_path = os.path.join(str(path), str(sub), "scheduler_config.json")
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(f"DDPMScheduler.from_pretrained: no local scheduler config {cfg_path} (models are read from disk only)")
        with open(cfg_path) as f:
            cfg = json.load(f)
        return _ddpm({**cfg, **kw}, cfg_path), None
    if target.startswith("diffusers.") and name == "DDPMScheduler":
        unknown = sorted(set(kw) - set(DDPM_DEFAULTS) - DDPM_SAMPLING_KEYS)
        if unknown:
            raise TypeError(f"DDPMScheduler.__init__() got unexpected keyword arguments {unknown}")
        return _ddpm(kw, "DDPMScheduler"), None
    if target.startswith("hcpdiff.noise") and name in ("ZeroTerminalScheduler", "PyramidNoiseScheduler"):
        if "base_scheduler" not in kw:
            raise ValueError(f"{name}: base_scheduler is required")
        base = kw.pop("base_scheduler")
        if name == "ZeroTerminalScheduler":
            if kw:
                raise TypeError(f"ZeroTerminalScheduler.__init__() got unexpected keyword arguments {sorted(kw)}")
            betas, pyramid = _resolve(base, inside_zero_terminal=True)
            return rescale_zero_terminal_snr(betas), pyramid
        if inside_zero_terminal:
            raise NotImplementedError(
                "ZeroTerminalScheduler around PyramidNoiseScheduler: the reference then rescales the wrapper's tables, not those of the "
                "DDPMScheduler whose add_noise runs, so x_t and the loss would use different tables; nest them as "
                "PyramidNoiseScheduler(ZeroTerminalScheduler(DDPMScheduler))")
        unknown = sorted(set(kw) - set(PYRAMID_DEFAULTS))
        if unknown:
            raise TypeError(f"PyramidNoiseScheduler.__init__() got unexpected keyword arguments {unknown}")
        opts = {**PYRAMID_DEFAULTS, **kw}
        if opts["resize_mode"] != "bilinear":
            raise NotImplementedError(f"PyramidNoiseScheduler resize_mode={opts['resize_mode']!r}: only 'bilinear'")
        level, step_size = int(opts["level"]), float(opts["step_size"])
        if not 1 <= level <= PYRAMID_MAX_LEVEL:
            raise ValueError(f"PyramidNoiseScheduler level={level}: 1 .. {PYRAMID_MAX_LEVEL}")
        if not step_size >= 1.0:
            raise ValueError(f"PyramidNoiseScheduler step_size={step_size}: must be >= 1 (a smaller ratio makes grids larger than the latent)")
        betas, inner = _resolve(base, inside_zero_terminal)
        if inner is not None:
            raise NotImplementedError("PyramidNoiseScheduler around another PyramidNoiseScheduler is not supported")
        return betas, {"level": level, "discount": float(opts["discount"]), "step_size": step_size}
    raise NotImplementedError(f"model.noise_scheduler._target_={target!r}: diffusers.DDPMScheduler (or .from_pretrained), "
                              "hcpdiff.noise.ZeroTerminalScheduler or hcpdiff.noise.PyramidNoiseScheduler")


def resolve(cfg, loss=None) -> NoiseSchedule:
    """`model.noise_scheduler` -> NoiseSchedule.  None gives SD1.x's table, `engine.ddpm_alphas_cumprod()`, bit for bit.  `loss`: the
    engine loss spec (None / 'mse' / {'type', 'gamma'}), checked with `check_loss`."""
    if isinstance(cfg, NoiseSchedule):
        sched = cfg
    elif cfg is None:
        from .engine import ddpm_alphas_cumprod
        sched = NoiseSchedule(ddpm_alphas_cumprod())
    else:
        betas, pyramid = _resolve(cfg)
        sched = NoiseSchedule(torch.cumprod(1.0 - betas, dim=0), pyramid)
    check_loss(sched, loss)
    return sched


def check_loss(sched: NoiseSchedule, loss) -> None:
    """EDMLoss weighs t by 1 / SNR(t): infinite where alphas_cumprod is 0 (zero terminal SNR at t = T-1)."""
    kind = loss if isinstance(loss, str) else (loss or {}).get("type")
    if kind in ("edm", "EDMLoss") and float(sched.alphas_cumprod.min()) == 0.0:
        raise ValueError("EDMLoss with a zero-terminal-SNR schedule (ZeroTerminalScheduler / rescale_betas_zero_snr): its weight is "
                         "infinite at t = T-1, where the SNR is 0")
