"""Generate tests/golden/ref_noise.pt from the UNMODIFIED reference noise schedulers (hcpdiff/noise/pyramid_noise.py,
zero_terminal.py, noise_base.py).

Run in a container that has the reference tree (the GPU machines do not):  python tests/golden/make_golden_noise.py

diffusers is not importable here, so a stub module provides the empty `SchedulerMixin` base the reference classes inherit, and a
stub base scheduler stands in for DDPMScheduler: it carries the betas / alphas / alphas_cumprod that ZeroTerminalScheduler
rewrites and records the noise PyramidNoiseScheduler hands to its add_noise.

  pyramid   per case: the inputs of PyramidNoiseScheduler.add_noise (the base noise as the seed of `base_noise`, plus its first
            values to check the regeneration), the (hn, wn) of every torch.randn call it made, the std it divided by, and at
            SAMPLES fixed flat indices the caller's noise tensor after the call (modified in place: the reference's loss target)
            and the normalised noise its base scheduler received.  `random.random` and `torch.randn` are patched to return the
            draws tests/noise_ref.py defines (the kernels' Philox draws) for the case's (seed, draw, group).
  zero_terminal  per beta schedule: the base betas and ZeroTerminalScheduler's float32 betas / alphas_cumprod.
"""
import os
import random
import sys
import types

import torch

REF = os.environ.get("HCP_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import noise_ref as N  # noqa: E402

# (B, H, W, level, discount, step_size, seed, draw, group)
CASES = [
    (1, 64, 64, 10, 0.9, 2.0, 11, 0, 0),
    (1, 128, 96, 10, 0.9, 2.0, 12, 5, 1),
    (3, 8, 8, 10, 0.5, 2.0, 13, 1, 0),
    (1, 64, 64, 1, 0.9, 2.0, 14, 0, 0),
    (3, 64, 64, 2, 0.5, 3.0, 15, 2, 2),
    (1, 128, 96, 10, 0.5, 1.0, 16, 3, 0),
    (3, 8, 8, 10, 0.9, 3.0, 17, (1 << 32) + 7, 1),
    (1, 8, 8, 10, 0.9, 1.0, (1 << 40) + 18, 9, 0),
]
SAMPLES = 2048         # elements recorded per case (the first and last element of the tensor included)
SCHEDULES = [("linear", 0.0001, 0.02), ("scaled_linear", 0.00085, 0.012), ("squaredcos_cap_v2", 0.0001, 0.02)]


def import_reference_noise():
    sys.dont_write_bytecode = True
    d = types.ModuleType("diffusers")
    d.SchedulerMixin = type("SchedulerMixin", (), {})
    sys.modules["diffusers"] = d
    pkg = types.ModuleType("hcpdiff")
    pkg.__path__ = [os.path.join(REF, "hcpdiff")]
    sys.modules["hcpdiff"] = pkg
    import hcpdiff.noise as noise
    return noise


class StubBase:
    """DDPMScheduler's tables and an add_noise that records what it is given."""

    def __init__(self, betas=None):
        if betas is not None:
            self.betas = betas
            self.alphas = 1.0 - betas
            self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.received = None

    def add_noise(self, original, noise, t):
        self.received = noise.clone()
        return original


def base_noise(B: int, H: int, W: int, seed: int) -> torch.Tensor:
    """The case's base N(0,1) noise [B, 4, H, W] (CPU generator: the same values wherever the tests run)."""
    return torch.randn((B, 4, H, W), generator=torch.Generator().manual_seed(seed))


def sample_index(n: int, seed: int) -> torch.Tensor:
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(seed + 1))[:SAMPLES - 2]
    return torch.cat([torch.tensor([0, n - 1]), idx]).sort().values


def pyramid_cases(noise):
    out = []
    for (B, H, W, level, discount, step_size, seed, draw, group) in CASES:
        base = base_noise(B, H, W, seed)
        levels = iter(range(1, level))
        sizes = []
        real_random, real_randn = random.random, torch.randn

        def fake_random():
            return N.uniform53(seed, draw, group, len(sizes) + 1)

        def fake_randn(b, c, hn, wn):
            i = next(levels)
            sizes.append((hn, wn))
            return torch.from_numpy(N.normals(seed, draw, group, i, b * c * hn * wn).reshape(b, c, hn, wn))

        stub = StubBase()
        sched = noise.PyramidNoiseScheduler(stub, level=level, discount=discount, step_size=step_size)
        caller = base.clone()
        random.random, torch.randn = fake_random, fake_randn
        try:
            sched.add_noise(torch.zeros_like(caller), caller, torch.zeros(B, dtype=torch.int64))
        finally:
            random.random, torch.randn = real_random, real_randn
        idx = sample_index(caller.numel(), seed)
        out.append({"B": B, "H": H, "W": W, "level": level, "discount": discount, "step_size": step_size, "seed": seed, "draw": draw,
                    "group": group, "noise_head": base.flatten()[:16].clone(), "sizes": sizes, "std": float(caller.std()),
                    "index": idx, "target": caller.flatten()[idx].clone(), "normalised": stub.received.flatten()[idx].clone()})
    return out


def zero_terminal_tables(noise):
    from hcp_diffusion_b200.noise import ddpm_betas
    out = {}
    for name, b0, b1 in SCHEDULES:
        betas = ddpm_betas(1000, b0, b1, name)
        stub = StubBase(betas.clone())
        noise.ZeroTerminalScheduler(stub)
        out[name] = {"beta_start": b0, "beta_end": b1, "betas_in": betas, "betas": stub.betas, "alphas_cumprod": stub.alphas_cumprod}
    return out


def main():
    noise = import_reference_noise()
    blob = {"pyramid": pyramid_cases(noise), "zero_terminal": zero_terminal_tables(noise)}
    path = os.path.join(HERE, "ref_noise.pt")
    torch.save(blob, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
