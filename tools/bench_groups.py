"""Time the training step with data groups on one GPU: `python tools/bench_groups.py [--steps K] [--warmup W]`.

Workloads (SD1.5 UNet, 512x512 = 64x64 latents, 77 x 768 text, synthetic weights and inputs):
  lora        LoRA r=8 on every attn1 / attn2 Linear, instance batch 4 (one group, `step_groups`)
  lora+class  the same with a prior-preservation class group of 1 carrying a per-pixel loss mask (DreamBooth.yaml's dataset_class)
  ft          full fine-tune of every UNet parameter, batch 16 (BASELINE config 3 shapes)
  ft4         full fine-tune, instance batch 4 (DreamBooth.yaml's dataset1)
  ft4+class   the same with a masked class group of 1 (DreamBooth.yaml's dataset_class)
(One UNet pass takes any number of images; the class group rides on DreamBooth.yaml's instance batch 4.)
One JSON line per workload: ms per step (CUDA events around K steps, each ending with the D2H read of the logged loss, as the
reference's loss.item()) and images/s counting every group's images, with the card's name and power limit read in the same run.
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

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import unet_ref as U  # noqa: E402   (synthetic weight / input generators)


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return name, power


def batches(sizes, masked, seed):
    out = []
    for g, B in enumerate(sizes):
        lat, noise, t, ehs = U.synthetic_batch(B, U.SD15, seed=seed + g)
        b = {"latents": lat.pin_memory(), "noise": noise.pin_memory(), "t": t.pin_memory(), "ehs": ehs.pin_memory()}
        if g in masked:
            b["mask"] = (torch.rand((B, 64, 64), generator=torch.Generator().manual_seed(seed + g)) * 5).pin_memory()
        out.append(b)
    return out


def run(kind, sizes, masked, steps, warmup, dev):
    torch.manual_seed(0)
    unet = UNet2DConditionModel()
    unet.load_state_dict(U.init_params(U.SD15, seed=0))
    unet = unet.to(dev).requires_grad_(False).eval()
    if kind == "ft":
        groups, _ = make_hcpdiff(unet, [{"lr": 1e-6, "layers": [""]}], None)
    else:
        groups, _ = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 8, "alpha": 1.0, "dropout": 0.0, "layers": [r"re:.*\.attn.?$"]}])
    step = LoraTrainStep(unet, groups, weight_decay=1e-2, max_grad_norm=1.0, use_cuda_graph=True, loss_weights=[1.0] * len(sizes))
    data = [batches(sizes, masked, 1234 + 10 * i) for i in range(2)]
    losses = []
    for i in range(warmup):
        losses.append(float(step.step_groups(data[i % 2])[-1].cpu()))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        losses.append(float(step.step_groups(data[i % 2])[-1].cpu()))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del step, unet, groups
    gc.collect()
    torch.cuda.empty_cache()
    return ms, losses


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", type=str, default="", help="comma-separated subset of lora, lora+class, ft, ft4, ft4+class")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_groups: needs a CUDA device (no CPU timing is reported)")
    dev = torch.device("cuda")
    _lib.check(_lib.lib().hcp_device_check(), "hcp_device_check")
    name, power = card()
    work = {"lora": ("lora", (4,), ()), "lora+class": ("lora", (4, 1), (1,)), "ft": ("ft", (16,), ()), "ft4": ("ft", (4,), ()),
            "ft4+class": ("ft", (4, 1), (1,))}
    chosen = [w for w in work if not args.only or w in args.only.split(",")]
    for w in chosen:
        kind, sizes, masked = work[w]
        ms, losses = run(kind, sizes, masked, args.steps, args.warmup, dev)
        images = sum(sizes)
        print(json.dumps({"workload": w, "group_batches": list(sizes), "masked_groups": list(masked), "steps": args.steps,
                          "warmup": args.warmup, "ms_per_step": round(ms, 3), "images_per_s": round(images * 1000.0 / ms, 2),
                          "last_loss": losses[-1], "finite": all(l == l for l in losses), "gpu": name, "power_limit_w": power}),
              flush=True)


if __name__ == "__main__":
    main()
