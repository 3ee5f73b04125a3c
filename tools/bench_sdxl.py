"""BASELINE config 4 on one H100: SDXL-base UNet (2.57 B parameters, random init), LoRA rank 16 on every attn / ff Linear and on the
resnet / sampler convolutions (locon), batch 2, 1024x1024 (128x128 latent), 77 tokens x 2048.  Prints one JSON line with the step
time.  Not the benchmark contract (bench.py measures config 2); a reference point for the SDXL rows of DESIGN.md.
`--full-ft` trains every parameter of the UNet instead (reference cfgs/train/examples/FT_sdxl.yaml), with `--optimizer adamw`,
`adafactor` (relative_step False, lr 1e-6, weight_decay 1e-3 as there), `lion` (lr 1e-6, weight_decay 1e-2 as the reference's
Lion_optimizer.yaml) or `adamw8bit` (bitsandbytes' AdamW8bit, weight_decay 1e-3 as cfgs/train/ft_adamw8bit_sdxl_synthetic.yaml);
the line then also gives the optimizer's own time per step.
`--lora-te` times, in the same run, the step above and then the same step with SDXL's two text encoders (CLIP-L + OpenCLIP-bigG,
full size, random init) in front, LoRA rank 4 on their self_attn + mlp layers (reference cfgs/train/examples/lora_sdxl.yaml's
lora_text_encoder item, clip_skip 1, no final norm): the line gives both step times, the card and its power limit.
`--full-te` does the same with every parameter of both text encoders trained instead (`text_encoder: [{lr: 1e-6, layers: ['']}]`,
reference cfgs/train/examples/fine-tuning.yaml), keys `*_full_te`.

  python tools/bench_sdxl.py [--batch 2] [--steps 5] [--no-locon] [--full-ft --optimizer adafactor|lion|adamw8bit] [--lora-te | --full-te]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import SDXLTextEncoder, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=2)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--latent", type=int, default=128)
ap.add_argument("--rank", type=int, default=16)
ap.add_argument("--no-locon", action="store_true")
ap.add_argument("--full-ft", action="store_true")
ap.add_argument("--optimizer", choices=("adamw", "adafactor", "lion", "adamw8bit"), default="adamw")
ap.add_argument("--lora-te", action="store_true")
ap.add_argument("--full-te", action="store_true")
args = ap.parse_args()
if (args.lora_te or args.full_te) and (args.full_ft or args.optimizer != "adamw"):
    ap.error("--lora-te / --full-te time the UNet LoRA step with AdamW")
if args.lora_te and args.full_te:
    ap.error("--lora-te and --full-te are two runs")


def random_init(module):
    """Timing only: fan-in scaled random weights, unit norm scales."""
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() > 1:
                fan_in = p[0].numel()
                p.normal_(0, fan_in ** -0.5)
            elif "norm" in name and name.endswith("weight"):
                p.fill_(1.0)
            else:
                p.zero_()


def time_steps(step, *inputs):
    for _ in range(3):
        step.step(*inputs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step.step(*inputs)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps


torch.manual_seed(0)
t0 = time.time()
with torch.device("meta"):
    unet = UNet2DConditionModel(sample_size=args.latent, block_out_channels=(320, 640, 1280), attention_head_dim=(5, 10, 20),
                                cross_attention_dim=2048, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                                up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                                transformer_layers_per_block=(1, 2, 10), use_linear_projection=True, addition_embed_type="text_time",
                                addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816)
unet = unet.to_empty(device="cuda")
random_init(unet)
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
elif args.optimizer == "lion":
    step = LoraTrainStep(unet, groups if args.full_ft else params, optimizer="lion", weight_decay=1e-2)
elif args.optimizer == "adamw8bit":
    step = LoraTrainStep(unet, groups if args.full_ft else params, optimizer="adamw8bit", weight_decay=1e-3)
else:
    step = LoraTrainStep(unet, groups if args.full_ft else params)
B, S = args.batch, args.latent
lat, noise = torch.randn(B, 4, S, S), torch.randn(B, 4, S, S)
t, ehs = torch.randint(0, 1000, (B,)), torch.randn(B, 77, 2048)
px = float(S * 8)
added = {"text_embeds": torch.randn(B, 1280), "time_ids": torch.tensor([[px, px, 0.0, 0.0, px, px]]).repeat(B, 1)}
ms = time_steps(step, lat, noise, t, ehs, added)
build_s = time.time() - t0
# the optimizer graph alone (clip + optimizer + EMA + zero_grad).  It ends by zeroing the gradient buffer, so these replays run on
# zero gradients (the same memory traffic as a real step) and move the parameters and optimizer state after the timed steps.
opt_reps = 5
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(opt_reps):
    step._graph_opt.replay()
e1.record()
torch.cuda.synchronize()
opt_ms = e0.elapsed_time(e1) / opt_reps
props = torch.cuda.get_device_properties(0)
out = {"workload": workload + f", bs={B}, {S * 8}x{S * 8}", "ms_per_step": ms, "images_per_s": B / ms * 1e3,
       "optimizer_ms": opt_ms, ("trained_params" if args.full_ft else "lora_params"): sum(p.numel() for p in params),
       "optimizer_state_bytes": step.optimizer_state_bytes, "launches_per_step": step.launches_per_step,
       "loss": float(step.loss.cpu()), "build_s": round(build_s, 1),
       "max_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "gpu": props.name}
if args.lora_te or args.full_te:
    # the same UNet and adapters, with SDXL's text encoders in front: ids [B, 2 x 77] (same words, bigG's chunk padded with id 0
    # after EOS), text_embeds from bigG's projected pooled row; the step above is released first
    del step
    torch.cuda.empty_cache()
    with torch.device("meta"):
        te = SDXLTextEncoder()
    te = te.to_empty(device="cuda")
    random_init(te)
    te.requires_grad_(False).eval()
    if args.full_te:
        te_groups, te_lora = make_hcpdiff(te, [{"lr": 1e-6, "layers": [""]}], None, default_lr=1e-5)
    else:
        te_groups, te_lora = make_hcpdiff(te, None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=1e-5)
    step_te = LoraTrainStep(unet, [{"params": params}] + te_groups, text_encoder=te, text_encoder_opts={"clip_skip": 1, "clip_final_norm": False})
    g = torch.Generator().manual_seed(1)
    n_words = torch.randint(5, 70, (B,), generator=g)
    ids = torch.full((B, 154), 49407, dtype=torch.int64)
    ids[:, 0] = ids[:, 77] = 49406
    for b in range(B):
        n = int(n_words[b])
        words = torch.randint(0, 49406, (n,), generator=g)
        ids[b, 1:1 + n] = ids[b, 78:78 + n] = words
        ids[b, 79 + n:] = 0
    ms_te = time_steps(step_te, lat, noise, t, ids, {"time_ids": added["time_ids"]})
    # forward GEMM FLOP per prompt of L = 77 tokens, from shapes: per layer 2 L (4 C^2 + 2 C F) (q, k, v, out_proj, fc1, fc2) over
    # the layers that run (clip_skip 1: 11 of clip_B's 12, all 32 of bigG's), plus bigG's projection of the pooled row
    L = 77
    gflop = {}
    for name, enc, n_layers in (("clip_B", te.clip_B, 11), ("clip_bigG", te.clip_bigG, 32)):
        C_, F_ = enc.config.hidden_size, enc.config.intermediate_size
        gflop[name] = n_layers * 2 * L * (4 * C_ * C_ + 2 * C_ * F_) / 1e9
    gflop["clip_bigG"] += 2 * 1280 * 1280 / 1e9
    sfx = "full_te" if args.full_te else "lora_te"
    out.update({f"ms_per_step_{sfx}": ms_te, f"images_per_s_{sfx}": B / ms_te * 1e3,
                f"te_{'trained' if args.full_te else 'lora'}_params": sum(p.numel() for g in te_groups for p in g["params"]),
                "te_forward_gemm_gflop_per_prompt": {k: round(v, 1) for k, v in gflop.items()},
                f"launches_per_step_{sfx}": step_te.launches_per_step, f"optimizer_state_bytes_{sfx}": step_te.optimizer_state_bytes,
                f"loss_{sfx}": float(step_te.loss.cpu()), "max_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)})
try:
    out["power_limit_w"] = float(subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                                capture_output=True, text=True, timeout=30).stdout.split()[0])
except (OSError, ValueError, IndexError, subprocess.SubprocessError):
    out["power_limit_w"] = None
print(json.dumps(out))
