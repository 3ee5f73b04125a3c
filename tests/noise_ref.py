"""float64 restatement of the pyramid noise kernels (include/hcp_b200.h: hcp_pyramid_plan, hcp_pyramid_noise) and of the noise
schedules, for the CPU and GPU tests.

The random numbers are those the kernels define, from tests/philox_ref.py: the level ratios r_i = 2 U + step_size (U a 53-bit double
from Philox counter (i, 0xFFFFFFFF, group, draw_lo)) and the level grids (Box-Muller on Philox counter (q, i, group, draw_lo) for
elements 4q .. 4q+3), key (seed_lo, seed_hi ^ draw_hi).  The sizes follow PyramidNoiseScheduler.add_noise
(hcpdiff/noise/pyramid_noise.py:25-31), the upsampling PyTorch's bilinear rule with align_corners=False (source index and weights
in fp32 as torch computes them, the source index with one fused multiply-add), the sum is in float64.
"""
import math

import numpy as np

from philox_ref import MASK, philox4x32_10

PLAN_TAG = 0xFFFFFFFF


def golden_base_noise(case):
    """The base noise of a tests/golden/ref_noise.pt pyramid case, regenerated from its seed (checked against its first values)."""
    import torch
    base = torch.randn((case["B"], 4, case["H"], case["W"]), generator=torch.Generator().manual_seed(case["seed"]))
    assert torch.equal(base.flatten()[:16], case["noise_head"]), "torch.randn no longer reproduces the golden's base noise"
    return base


def _key(seed: int, draw: int):
    return seed & 0xFFFFFFFF, ((seed >> 32) ^ (draw >> 32)) & 0xFFFFFFFF


def uniform53(seed: int, draw: int, group: int, level: int) -> float:
    """U of level i (1-based) for one data group: ((w0 >> 5) 2^26 + (w1 >> 6)) / 2^53, as Python's random.random builds it."""
    w = philox4x32_10(level, PLAN_TAG, group, draw & 0xFFFFFFFF, *_key(seed, draw))
    return ((int(w[0]) >> 5) * 67108864.0 + (int(w[1]) >> 6)) / 9007199254740992.0


def plan(seed: int, draw: int, group: int, level: int, step_size: float, H: int, W: int):
    """[(hn_i, wn_i)] for i = 1 .. n, the sizes pyramid_noise.py:26-31 computes from the ratios above."""
    sizes = []
    for i in range(1, level):
        r = uniform53(seed, draw, group, i) * 2 + step_size
        wn, hn = max(1, int(W / (r ** i))), max(1, int(H / (r ** i)))
        sizes.append((hn, wn))
        if wn == 1 or hn == 1:
            break
    return sizes


def normals(seed: int, draw: int, group: int, level: int, n: int) -> np.ndarray:
    """float32 [n]: the first n elements of the group's level-i grid in torch.randn's flat order."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    w = philox4x32_10(q & MASK, level, group, draw & 0xFFFFFFFF, *_key(seed, draw))
    out = np.empty((q.size, 4), dtype=np.float64)
    for j in (0, 2):
        u1 = (w[j].astype(np.float64) + 1.0) * 2.0 ** -32
        u2 = w[j + 1].astype(np.float64) * 2.0 ** -32
        rad = np.sqrt(-2.0 * np.log(u1))
        out[:, j], out[:, j + 1] = rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)
    return out.reshape(-1)[:n].astype(np.float32)


def _weights(n_in: int, n_out: int):
    scale = np.float32(n_in) / np.float32(n_out)
    dst = np.arange(n_out, dtype=np.float32) + np.float32(0.5)
    # fused multiply-add, one rounding to fp32 (the fp64 product of two fp32 values is exact), as torch's compiled kernels do
    src = np.maximum((np.float64(scale) * dst.astype(np.float64) - 0.5).astype(np.float32), np.float32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    lam = np.clip(src - i0.astype(np.float32), 0, 1).astype(np.float64)
    i1 = i0 + (i0 < n_in - 1)
    return i0, i1, 1.0 - lam, lam


def bilinear(grid: np.ndarray, H: int, W: int) -> np.ndarray:
    """F.interpolate(grid [..., hn, wn], (H, W), mode='bilinear', align_corners=False) in float64."""
    y0, y1, ly0, ly1 = _weights(grid.shape[-2], H)
    x0, x1, lx0, lx1 = _weights(grid.shape[-1], W)
    g = grid.astype(np.float64)
    top = g[..., y0, :][..., x0] * lx0 + g[..., y0, :][..., x1] * lx1
    bot = g[..., y1, :][..., x0] * lx0 + g[..., y1, :][..., x1] * lx1
    return top * ly0[:, None] + bot * ly1[:, None]


def pyramid(noise: np.ndarray, sizes, discount: float, seed: int, draw: int, group: int):
    """(target, inv_std) of one data group: noise [b, c, H, W] + sum_i bilinear(grid_i) discount^i, and 1 / its unbiased std."""
    b, c, H, W = noise.shape
    out = noise.astype(np.float64).copy()
    for i, (hn, wn) in enumerate(sizes, start=1):
        grid = normals(seed, draw, group, i, b * c * hn * wn).reshape(b, c, hn, wn)
        out += bilinear(grid, H, W) * float(np.float32(discount ** i))
    return out, 1.0 / out.std(ddof=1)


def ddpm_betas(T: int, beta_start: float, beta_end: float, schedule: str) -> np.ndarray:
    """DDPMScheduler's betas in float64 (diffusers' linear, scaled_linear, squaredcos_cap_v2)."""
    if schedule == "linear":
        return np.linspace(beta_start, beta_end, T)
    if schedule == "scaled_linear":
        return np.linspace(beta_start ** 0.5, beta_end ** 0.5, T) ** 2

    def alpha_bar(t):
        return math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
    return np.array([min(1 - alpha_bar((i + 1) / T) / alpha_bar(i / T), 0.999) for i in range(T)])


def zero_terminal(betas: np.ndarray) -> np.ndarray:
    """arXiv 2305.08891 Algorithm 1 in float64: betas rescaled so that alphas_cumprod[T-1] == 0."""
    s = np.sqrt(np.cumprod(1.0 - betas))
    s = (s - s[-1]) * s[0] / (s[0] - s[-1])
    a = s ** 2
    return 1.0 - np.concatenate([a[:1], a[1:] / a[:-1]])
