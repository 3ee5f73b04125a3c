"""What `model.gradient_checkpointing` costs and which batches it opens, on one GPU: `python tools/bench_ckpt.py [--steps K]`.

In one process, for each workload and batch, the step is timed with the flag off and then on (CUDA events around K captured steps
after a warm-up, each step ending with the D2H read of the logged loss), with `max_memory_allocated` of that leg:
  sd15_lora   SD1.5 UNet, LoRA r=8 on every attn1 / attn2 Linear (BASELINE config 2), 512x512, batch 4 / 16 / 32 / 64
  sdxl_locon  SDXL-base UNet, LoRA r=16 on attn / ff and the resnet / sampler convolutions (config 4), 1024x1024, batch 2 / 4 / 8 / 16
  sdxl_ft     SDXL-base UNet full fine-tune with Lion and with AdamW8bit, 1024x1024, batch 1, 2, 3, ... until the leg no longer fits
A leg that does not fit in the card's memory is reported as {"fits": false}; a flag-off leg that failed is not retried at a larger
batch.  Synthetic weights and inputs (fan-in scaled random init).  One JSON line per leg, then one line with the card's name and power
limit read in the same run.
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

from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--only", choices=("sd15_lora", "sdxl_locon", "sdxl_ft"), default=None)
args = ap.parse_args()


def random_init(module):
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() > 1:
                p.normal_(0, p[0].numel() ** -0.5)
            elif "norm" in name and name.endswith("weight"):
                p.fill_(1.0)
            else:
                p.zero_()


def make_unet(xl: bool):
    with torch.device("meta"):
        if xl:
            u = UNet2DConditionModel(sample_size=128, block_out_channels=(320, 640, 1280), attention_head_dim=(5, 10, 20),
                                     cross_attention_dim=2048, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                                     up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                                     transformer_layers_per_block=(1, 2, 10), use_linear_projection=True, addition_embed_type="text_time",
                                     addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816)
        else:
            u = UNet2DConditionModel()
    u = u.to_empty(device="cuda")
    random_init(u)
    return u.requires_grad_(False).eval()


def inputs(B, xl):
    S, ctx = (128, 2048) if xl else (64, 768)
    g = torch.Generator().manual_seed(B)
    lat, noise = torch.randn(B, 4, S, S, generator=g), torch.randn(B, 4, S, S, generator=g)
    t, ehs = torch.randint(0, 1000, (B,), generator=g), torch.randn(B, 77, ctx, generator=g)
    if not xl:
        return (lat, noise, t, ehs)
    px = float(S * 8)
    return (lat, noise, t, ehs, {"text_embeds": torch.randn(B, 1280, generator=g),
                                 "time_ids": torch.tensor([[px, px, 0.0, 0.0, px, px]]).repeat(B, 1)})


def leg(name, unet, make_step, B, xl, on):
    unet.gradient_checkpointing = on
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    out = {"workload": name, "batch": B, "checkpointing": on}
    step = None
    try:
        step = make_step()
        x = inputs(B, xl)
        for _ in range(2):
            float(step.step(*x).cpu())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            loss = float(step.step(*x).cpu())
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        out.update({"fits": True, "ms_per_step": round(ms, 2), "images_per_s": round(B / ms * 1e3, 2), "loss": loss,
                    "max_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)})
    except torch.cuda.OutOfMemoryError:
        out.update({"fits": False})
    finally:
        del step
        unet.gradient_checkpointing = False
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)
    return out["fits"]


torch.manual_seed(0)
if args.only in (None, "sd15_lora"):
    unet = make_unet(False)
    groups, _ = make_hcpdiff(unet, None, [{"rank": 8, "dropout": 0.0, "lr": 1e-4, "layers": [r"re:.*\.attn.?$"]}])
    params = [p for g in groups for p in g["params"]]
    for B in (4, 16, 32, 64):
        for on in (False, True):
            leg("sd15_lora_r8_512", unet, lambda: LoraTrainStep(unet, params, lr=1e-4), B, False, on)
    del unet, groups, params
if args.only in (None, "sdxl_locon"):
    unet = make_unet(True)
    layers = [r"re:.*\.attn.?$", r"re:.*\.ff$", r"re:.*\.resnets\.\d+\.conv[12]$", r"re:.*\.conv_shortcut$", r"re:.*samplers\.0\.conv$"]
    groups, _ = make_hcpdiff(unet, None, [{"rank": 16, "dropout": 0.0, "layers": layers}])
    params = [p for g in groups for p in g["params"]]
    off_fits = True
    for B in (2, 4, 8, 16):
        for on in (False, True):
            if on or off_fits:
                fits = leg("sdxl_lora_r16_locon_1024", unet, lambda: LoraTrainStep(unet, params), B, True, on)
                off_fits = fits if not on else off_fits
    del unet, groups, params
if args.only in (None, "sdxl_ft"):
    unet = make_unet(True)
    groups, _ = make_hcpdiff(unet, [{"lr": 1e-6, "layers": [""]}], None)
    for opt, kw in (("lion", {"weight_decay": 1e-2}), ("adamw8bit", {"weight_decay": 1e-3})):
        for on in (False, True):
            B = 1
            while leg(f"sdxl_full_ft_{opt}_1024", unet, lambda: LoraTrainStep(unet, groups, optimizer=opt, **kw), B, True, on):
                B += 1
    del unet, groups

props = torch.cuda.get_device_properties(0)
info = {"gpu": props.name, "total_mem_gb": round(props.total_memory / 2 ** 30, 1)}
try:
    info["power_limit_w"] = float(subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                                 capture_output=True, text=True, timeout=30).stdout.split()[0])
except (OSError, ValueError, IndexError, subprocess.SubprocessError):
    info["power_limit_w"] = None
print(json.dumps(info), flush=True)
