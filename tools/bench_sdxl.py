"""BASELINE config 4 on one H100: SDXL-base UNet (2.57 B parameters, random init), LoRA rank 16 on every attn / ff Linear and on the
resnet / sampler convolutions (locon), batch 2, 1024x1024 (128x128 latent), 77 tokens x 2048.  Prints one JSON line with the step
time.  Not the benchmark contract (bench.py measures config 2); a reference point for the SDXL rows of DESIGN.md.
`--full-ft` trains every parameter of the UNet instead (reference cfgs/train/examples/FT_sdxl.yaml), with `--optimizer adamw` or
`adafactor` (relative_step False, lr 1e-6, weight_decay 1e-3 as there); the line then also gives the optimizer's own time per step.

  python tools/bench_sdxl.py [--batch 2] [--steps 5] [--no-locon] [--full-ft --optimizer adafactor]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=2)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--latent", type=int, default=128)
ap.add_argument("--rank", type=int, default=16)
ap.add_argument("--no-locon", action="store_true")
ap.add_argument("--full-ft", action="store_true")
ap.add_argument("--optimizer", choices=("adamw", "adafactor"), default="adamw")
args = ap.parse_args()

torch.manual_seed(0)
t0 = time.time()
with torch.device("meta"):
    unet = UNet2DConditionModel(sample_size=args.latent, block_out_channels=(320, 640, 1280), attention_head_dim=(5, 10, 20),
                                cross_attention_dim=2048, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                                up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                                transformer_layers_per_block=(1, 2, 10), use_linear_projection=True, addition_embed_type="text_time",
                                addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816)
unet = unet.to_empty(device="cuda")
with torch.no_grad():
    for name, p in unet.named_parameters():           # timing only: fan-in scaled random weights, unit norm scales
        if p.dim() > 1:
            fan_in = p[0].numel()
            p.normal_(0, fan_in ** -0.5)
        elif "norm" in name and name.endswith("weight"):
            p.fill_(1.0)
        else:
            p.zero_()
unet.requires_grad_(False).eval()
if args.full_ft:
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-6, "layers": [""]}], None)
    workload = f"SDXL-base UNet full fine-tune, {args.optimizer}"
else:
    layers = [r"re:.*\.attn.?$", r"re:.*\.ff$"]
    if not args.no_locon:
        layers += [r"re:.*\.resnets\.\d+\.conv[12]$", r"re:.*\.conv_shortcut$", r"re:.*samplers\.0\.conv$"]
    groups, lora = make_hcpdiff(unet, None, [{"rank": args.rank, "dropout": 0.0, "layers": layers}])
    workload = f"SDXL-base UNet LoRA r={args.rank} attn+ff" + ("" if args.no_locon else "+conv (locon)")
params = [p for g in groups for p in g["params"]]
if args.optimizer == "adafactor":
    step = LoraTrainStep(unet, groups, optimizer="adafactor", optimizer_kwargs={"relative_step": False, "weight_decay": 1e-3})
else:
    step = LoraTrainStep(unet, groups if args.full_ft else params)
B, S = args.batch, args.latent
lat, noise = torch.randn(B, 4, S, S), torch.randn(B, 4, S, S)
t, ehs = torch.randint(0, 1000, (B,)), torch.randn(B, 77, 2048)
px = float(S * 8)
added = {"text_embeds": torch.randn(B, 1280), "time_ids": torch.tensor([[px, px, 0.0, 0.0, px, px]]).repeat(B, 1)}
for _ in range(3):
    step.step(lat, noise, t, ehs, added)
torch.cuda.synchronize()
build_s = time.time() - t0
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.steps):
    step.step(lat, noise, t, ehs, added)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / args.steps
# the optimizer graph alone (clip + optimizer + EMA + zero_grad).  It ends by zeroing the gradient buffer, so these replays run on
# zero gradients (the same memory traffic as a real step) and move the parameters and optimizer state after the timed steps.
opt_reps = 5
e0.record()
for _ in range(opt_reps):
    step._graph_opt.replay()
e1.record()
torch.cuda.synchronize()
opt_ms = e0.elapsed_time(e1) / opt_reps
props = torch.cuda.get_device_properties(0)
print(json.dumps({"workload": workload + f", bs={B}, {S * 8}x{S * 8}", "ms_per_step": ms, "images_per_s": B / ms * 1e3,
                  "optimizer_ms": opt_ms, ("trained_params" if args.full_ft else "lora_params"): sum(p.numel() for p in params),
                  "optimizer_state_bytes": step.optimizer_state_bytes, "launches_per_step": step.launches_per_step,
                  "loss": float(step.loss.cpu()), "build_s": round(build_s, 1),
                  "max_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "gpu": props.name}))
