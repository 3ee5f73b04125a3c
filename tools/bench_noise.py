"""Cost of pyramid noise (`model.noise_scheduler: PyramidNoiseScheduler(ZeroTerminalScheduler(DDPMScheduler))`) on one GPU:
`python tools/bench_noise.py [--steps K] [--warmup W] [--rounds R] [--no-sdxl]`.

Step workloads (synthetic weights and inputs, CUDA graphs, MSE loss), each timed with the SD1.x DDPM table (no scheduler) and with
the pyramid, alternated R times:
  sd15   SD1.5 UNet, LoRA r=8 on every attn1 / attn2 Linear, batch 4, 512x512 (64x64 latent): bench.py's config 2 shapes
  sdxl   SDXL-base UNet (random init), LoRA r=16 on every attn / ff Linear, batch 2, 1024x1024 (128x128 latent)
Kernel workloads: plan + pyramid sum + scaled add_noise of one micro-step (`ops.PyramidNoise.add_noise`, level 10, discount 0.9,
step_size 2) on [4, 4, 64, 64] and [2, 4, 128, 128], CUDA events around 200 launches after 20 warm-up launches.
One JSON line per measurement, with the card's name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hcp_diffusion_b200 import _lib, noise  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.ops import PyramidNoise  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402   (synthetic weight / input generators)

PZ = {"_target_": "hcpdiff.noise.PyramidNoiseScheduler", "level": 10, "discount": 0.9, "step_size": 2.0,
      "base_scheduler": {"_target_": "hcpdiff.noise.ZeroTerminalScheduler",
                         "base_scheduler": {"_target_": "diffusers.DDPMScheduler", "beta_start": 0.00085, "beta_end": 0.012,
                                            "beta_schedule": "scaled_linear"}}}


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return name, power


def random_init(module):
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() > 1:
                p.normal_(0, p[0].numel() ** -0.5)
            elif "norm" in name and name.endswith("weight"):
                p.fill_(1.0)
            else:
                p.zero_()


def build(kind):
    torch.manual_seed(0)
    if kind == "sd15":
        unet = UNet2DConditionModel()
        unet.load_state_dict(U.init_params(U.SD15, seed=0))
        unet = unet.cuda()
        layers, rank, B, S, ctx = [r"re:.*\.attn.?$"], 8, 4, 64, 768
    else:
        with torch.device("meta"):
            unet = UNet2DConditionModel(sample_size=128, block_out_channels=(320, 640, 1280), attention_head_dim=(5, 10, 20),
                                        cross_attention_dim=2048, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                                        up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                                        transformer_layers_per_block=(1, 2, 10), use_linear_projection=True, addition_embed_type="text_time",
                                        addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816)
        unet = unet.to_empty(device="cuda")
        random_init(unet)
        layers, rank, B, S, ctx = [r"re:.*\.attn.?$", r"re:.*\.ff$"], 16, 2, 128, 2048
    unet.requires_grad_(False).eval()
    groups, _ = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": rank, "alpha": 1.0, "dropout": 0.0, "layers": layers}])
    g = torch.Generator().manual_seed(1)
    inputs = [torch.randn((B, 4, S, S), generator=g), torch.randn((B, 4, S, S), generator=g), torch.randint(0, 1000, (B,), generator=g),
              torch.randn((B, 77, ctx), generator=g)]
    if kind == "sdxl":
        px = float(S * 8)
        inputs.append({"text_embeds": torch.randn((B, 1280), generator=g), "time_ids": torch.tensor([[px, px, 0.0, 0.0, px, px]]).repeat(B, 1)})
    return unet, groups, [x.pin_memory() if torch.is_tensor(x) else {k: v.pin_memory() for k, v in x.items()} for x in inputs], B, S


def time_step(kind, scheduler, steps, warmup):
    unet, groups, inputs, B, S = build(kind)
    step = LoraTrainStep(unet, groups, use_cuda_graph=True, noise_scheduler=scheduler)
    for _ in range(warmup):
        float(step.step(*inputs).cpu())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = float(step.step(*inputs).cpu())                  # the reference's loss.item() every step
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    launches = step.launches_per_step
    del step, unet, groups
    gc.collect()
    torch.cuda.empty_cache()
    return ms, launches, loss, B, S


def time_kernels(B, S, reps=200):
    pn = PyramidNoise(10, 0.9, 2.0, "cuda", seed=1)
    acp = noise.resolve(PZ).alphas_cumprod.cuda()
    x0, base = torch.randn((B, 4, S, S), device="cuda"), torch.randn((B, 4, S, S), device="cuda")
    t = torch.randint(0, 1000, (B,), device="cuda")
    for _ in range(20):
        pn.add_noise(x0, base, t, acp, (B,))
        pn.advance()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        pn.add_noise(x0, base, t, acp, (B,))
        pn.advance()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1000.0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-sdxl", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_noise: needs a CUDA device (no CPU timing is reported)")
    _lib.check(_lib.lib().hcp_device_check(), "hcp_device_check")
    name, power = card()
    for B, S in ((4, 64), (2, 128)):
        us = time_kernels(B, S)
        print(json.dumps({"measure": "pyramid kernels per micro-step (plan + sum + scaled add_noise, incl. the counter advance)",
                          "shape": [B, 4, S, S], "us_per_call": round(us, 2), "gpu": name, "power_limit_w": power}), flush=True)
    for kind in ("sd15",) + (() if args.no_sdxl else ("sdxl",)):
        for r in range(args.rounds if kind == "sd15" else 1):
            for label, sched in (("ddpm", None), ("pyramid", PZ)):
                ms, launches, loss, B, S = time_step(kind, sched, args.steps, args.warmup)
                print(json.dumps({"measure": "step", "workload": kind, "noise": label, "round": r, "batch": B, "latent": S,
                                  "steps": args.steps, "ms_per_step": round(ms, 3), "launches_per_step": launches, "last_loss": loss,
                                  "gpu": name, "power_limit_w": power}), flush=True)


if __name__ == "__main__":
    main()
