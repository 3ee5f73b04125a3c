"""Restatement of bitsandbytes.optim.AdamW8bit (blockwise 8-bit Adam moments) -- test infrastructure.

Each rule restates one bitsandbytes function:

  * `Optimizer2State.init_state` (optim_bits forced to 8): a parameter with fewer than `min_8bit_size` elements keeps fp32 `state1` /
    `state2` (zeros); every other one keeps uint8 `state1` / `state2` (zeros) with `qmap1` the signed and `qmap2` the unsigned
    dynamic map, and fp32 `absmax1` / `absmax2` (zeros), one per 256-element block from the tensor's first element (the last block
    may be partial).  `Optimizer2State.update_step`: `step` += 1, then the 8-bit or the 32-bit update below.
  * `functional.create_dynamic_map(signed=True / False)`: hcp_diffusion_b200.adamw8bit.create_dynamic_map, computed in torch's fp32
    exactly as there.
  * `optimizer_update_8bit_blockwise` / `kOptimizerStatic8bit2StateBlockwise`, per element of a block, in fp32:
      a non-finite g: s1 = s2 = 0, p unchanged;  otherwise g' = g * gnorm_scale,
      s2 = map2[c2] absmax2;  s2 = s2 b2 + ((1 - b2) g') g';   s1 = map1[c1] absmax1;  s1 = s1 b1 + (1 - b1) g'
      absmax_new = max |s| over the block (after the update)
      p = p + step_size s1 / (sqrt(s2) + eps corr2),  step_size = -lr corr2 / corr1,  corr1 = 1 - b1^t,  corr2 = sqrt(1 - b2^t)
      if wd > 0: p = p (1 - lr wd)            (weight decay after the step; torch's AdamW decays first)
      c = quantize(s / absmax_new) with `quantize_2D`'s binary search (below); for the first moment, if the sign bit of map1[c]
      differs from s1's, c moves one step toward s1's sign (c + 1 when s1 > 0, else c - 1).
  * `optimizer_update_32bit` / `kOptimizer32bit2State` (ADAM): the same moment and parameter update on fp32 m, v, with no
    non-finite guard (a non-finite g propagates into m, v and p, as it does there and in torch's AdamW).

quantize_2D: pivot = 127, lower_pivot = 0, upper_pivot = 255, lower = -1 (signed) or 0, upper = 1; val = map[127]; for i in 64, 32,
.., 1: if x > val: lower_pivot, lower = pivot, val; pivot += i, else upper_pivot, upper = pivot, val; pivot -= i; val = map[pivot].
Then if x > val: upper_pivot if x > (upper + val) * 0.5 else pivot; otherwise lower_pivot if x < (lower + val) * 0.5 else pivot.
That is the nearest map entry, and an exact midpoint goes to the last probed entry (`pivot`).

Choices where bitsandbytes leaves it open, which the kernel makes too:
  * every operation above is rounded to fp32 on its own (no fused multiply-add), so the result is reproducible bit for bit;
  * an all-zero block (absmax_new = 0) encodes x = 0 for each element (bitsandbytes divides 0 by 0 there); it decodes to 0 either
    way, since every code of the block is multiplied by the scale 0;
  * `gnorm_scale` is the engine's clip factor times its grad_scale (bitsandbytes' percentile clipping, which would set it, is
    not implemented; the reference loop clips the gradients in place before the step, so it passes 1).

`use_adamw8bit` puts the optimizer into oracle.step_ref.ReferenceLoop in place of AdamW (clip_grad_norm_, accumulation, DDP
averaging and EMA as there).
"""
from __future__ import annotations

import numpy as np
import torch

from hcp_diffusion_b200.adamw8bit import BLOCK, create_dynamic_map
from oracle import step_ref as S

F32 = np.float32
MAP1 = create_dynamic_map(True).numpy()
MAP2 = create_dynamic_map(False).numpy()


def quantize(code: np.ndarray, x: np.ndarray, signed: bool) -> np.ndarray:
    """quantize_2D over an fp32 array: codes (int64) of the nearest entries of the sorted fp32 `code`."""
    x = np.asarray(x, dtype=F32)
    pivot = np.full(x.shape, 127, dtype=np.int64)
    lo_p, up_p = np.zeros_like(pivot), np.full_like(pivot, 255)
    lower, upper = np.full(x.shape, -1.0 if signed else 0.0, dtype=F32), np.ones(x.shape, dtype=F32)
    val = code[pivot]
    i = 64
    while i > 0:
        gt = x > val
        lo_p, lower = np.where(gt, pivot, lo_p), np.where(gt, val, lower)
        up_p, upper = np.where(gt, up_p, pivot), np.where(gt, upper, val)
        pivot = np.where(gt, pivot + i, pivot - i)
        val = code[pivot]
        i >>= 1
    gt = x > val
    hi_mid = ((upper + val).astype(F32) * F32(0.5)).astype(F32)
    lo_mid = ((lower + val).astype(F32) * F32(0.5)).astype(F32)
    return np.where(gt, np.where(x > hi_mid, up_p, pivot), np.where(x < lo_mid, lo_p, pivot))


def midpoint_distance(code: np.ndarray, x: np.ndarray) -> np.ndarray:
    """|x - m| over the nearest midpoint m of adjacent entries of `code`, in fp32 ulps of x (for the near-tie count)."""
    x = np.asarray(x, dtype=F32)
    mids = ((code[:-1] + code[1:]).astype(F32) * F32(0.5)).astype(F32)
    k = np.clip(np.searchsorted(mids, x), 1, len(mids) - 1)
    d = np.minimum(np.abs(x.astype(np.float64) - mids[k - 1]), np.abs(x.astype(np.float64) - mids[k]))
    return d / np.spacing(np.maximum(np.abs(x), F32(1e-30))).astype(np.float64)


def coefficients(lr, beta1, beta2, eps, wd, step):
    """fp32 (step_size, eps corr2, 1 - b1, 1 - b2, 1 - lr wd) of step `step`, each rounded as the kernel rounds it."""
    lr, b1, b2, eps, wd = (F32(v) for v in (lr, beta1, beta2, eps, wd))
    t = F32(step)
    corr1 = F32(F32(1.0) - F32(np.power(b1, t)))
    corr2 = F32(np.sqrt(F32(F32(1.0) - F32(np.power(b2, t)))))
    step_size = F32(F32(-lr * corr2) / corr1)
    return step_size, F32(eps * corr2), F32(F32(1.0) - b1), F32(F32(1.0) - b2), F32(F32(1.0) - F32(lr * wd))


def update_moments(s1, s2, g, gs, b1, b2, omb1, omb2, guard):
    """New (s1, s2, finite mask) from fp32 moments and raw gradients; `guard`: the 8-bit path's non-finite rule."""
    fin = np.isfinite(g) if guard else np.ones(g.shape, dtype=bool)
    with np.errstate(all="ignore"):
        gv = (g * F32(gs)).astype(F32)
        n2 = ((s2 * F32(b2)).astype(F32) + ((omb2 * gv).astype(F32) * gv).astype(F32)).astype(F32)
        n1 = ((s1 * F32(b1)).astype(F32) + (omb1 * gv).astype(F32)).astype(F32)
    return np.where(fin, n1, F32(0)), np.where(fin, n2, F32(0)), fin


def update_param(p, s1, s2, fin, step_size, eps_c, wd, decay):
    with np.errstate(all="ignore"):
        q = (s1 / (np.sqrt(s2).astype(F32) + eps_c).astype(F32)).astype(F32)
        w = (p + (step_size * q).astype(F32)).astype(F32)
        if F32(wd) > 0:
            w = (w * decay).astype(F32)
    return np.where(fin, w, p)


def block_max(a: np.ndarray, n: int) -> np.ndarray:
    nb = -(-n // BLOCK)
    pad = np.zeros(nb * BLOCK, dtype=F32)
    pad[:n] = np.abs(a)
    return pad.reshape(nb, BLOCK).max(axis=1)


def step_8bit(p, g, c1, c2, am1, am2, hyper, step, gs=1.0):
    """One blockwise 8-bit step of one tensor (flat fp32 p, g; uint8 c1, c2; fp32 absmax per block): returns (p, c1, c2, am1, am2,
    s1, s2) with s1 / s2 the updated moments before re-encoding."""
    lr, b1, b2, eps, wd = hyper
    step_size, eps_c, omb1, omb2, decay = coefficients(lr, b1, b2, eps, wd, step)
    n = p.size
    blk = np.arange(n) // BLOCK
    s1 = (MAP1[c1] * am1[blk]).astype(F32)
    s2 = (MAP2[c2] * am2[blk]).astype(F32)
    s1, s2, fin = update_moments(s1, s2, g, gs, b1, b2, omb1, omb2, True)
    n1, n2 = block_max(s1, n), block_max(s2, n)
    p = update_param(p, s1, s2, fin, step_size, eps_c, wd, decay)
    x1 = np.where(n1[blk] > 0, s1 / np.where(n1[blk] > 0, n1[blk], F32(1)), F32(0)).astype(F32)
    x2 = np.where(n2[blk] > 0, s2 / np.where(n2[blk] > 0, n2[blk], F32(1)), F32(0)).astype(F32)
    k1 = quantize(MAP1, x1, True)
    flip = np.signbit(MAP1[k1]) != np.signbit(s1)
    k1 = np.where(flip, (k1 + np.where(s1 > 0, 1, -1)) & 255, k1)
    k2 = quantize(MAP2, x2, False)
    return p, k1.astype(np.uint8), k2.astype(np.uint8), n1, n2, s1, s2


def step_32bit(p, g, m, v, hyper, step, gs=1.0):
    """One fp32-state step of one tensor: returns (p, m, v)."""
    lr, b1, b2, eps, wd = hyper
    step_size, eps_c, omb1, omb2, decay = coefficients(lr, b1, b2, eps, wd, step)
    m, v, fin = update_moments(m, v, g, gs, b1, b2, omb1, omb2, False)
    return update_param(p, m, v, fin, step_size, eps_c, wd, decay), m, v


class AdamW8bit(torch.optim.Optimizer):
    """bitsandbytes.optim.AdamW8bit on CPU tensors (the state keeps bitsandbytes' names)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, min_8bit_size=4096):
        super().__init__(params, {"lr": lr, "betas": tuple(betas), "eps": eps, "weight_decay": weight_decay})
        self.min_8bit_size = min_8bit_size

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            hyper = (group["lr"], group["betas"][0], group["betas"][1], group["eps"], group["weight_decay"])
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                n = p.numel()
                if not st:
                    st["step"] = 0
                    if n < self.min_8bit_size:
                        st["state1"], st["state2"] = np.zeros(n, F32), np.zeros(n, F32)
                    else:
                        nb = -(-n // BLOCK)
                        st["state1"], st["state2"] = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
                        st["absmax1"], st["absmax2"] = np.zeros(nb, F32), np.zeros(nb, F32)
                st["step"] += 1
                pv = p.detach().cpu().numpy().reshape(-1).astype(F32)
                gv = p.grad.detach().cpu().numpy().reshape(-1).astype(F32)
                if "absmax1" in st:
                    pn, st["state1"], st["state2"], st["absmax1"], st["absmax2"], _, _ = step_8bit(
                        pv, gv, st["state1"], st["state2"], st["absmax1"], st["absmax2"], hyper, st["step"])
                else:
                    pn, st["state1"], st["state2"] = step_32bit(pv, gv, st["state1"], st["state2"], hyper, st["step"])
                p.copy_(torch.from_numpy(pn).view_as(p))


def use_adamw8bit(ref: S.ReferenceLoop, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, min_8bit_size=4096) -> S.ReferenceLoop:
    """Replace the reference loop's AdamW by AdamW8bit over the same parameter groups and learning rates."""
    ref.opt = AdamW8bit([{"params": g["params"], "lr": g["lr"]} for g in ref.opt.param_groups], lr=ref.opt.defaults["lr"], betas=betas,
                        eps=eps, weight_decay=weight_decay, min_8bit_size=min_8bit_size)
    return ref
