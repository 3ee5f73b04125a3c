"""The text encoder's share of a training step on one GPU: SD1.5 (UNet and CLIP-L at full size, random init), batch 4, 512x512
(64x64 latent), 77-token prompts (BOS, random words, EOS padding), AdamW, CUDA graphs.  Five legs, each built fresh and timed in
the same process:
  unet_lora                 UNet LoRA rank 8 on attn + ff (lora_te_sd15_synthetic.yaml's lora_unet item), precomputed text embedding
  unet_lora+te_lora         the same with the text encoder in front, LoRA rank 4 on self_attn + mlp (its lora_text_encoder item)
  unet_lora+te_full         the same with every text-encoder parameter trained (fine-tuning.yaml's `text_encoder: [{layers: ['']}]`)
  unet_full                 every UNet parameter trained (DreamBooth.yaml's `unet:` item), precomputed text embedding
  unet_full+te_full         the same with every text-encoder parameter trained (dreambooth_te_sd15_synthetic.yaml)
Per leg: ms per step (CUDA events around `--steps` steps after `--warmup`), images/s, peak allocated memory of the leg and the
optimizer-state bytes; the card name and its power limit are read in the same run.  Prints one JSON line.

  python tools/bench_te.py [--batch 4] [--steps 10] [--warmup 3] [--legs unet_lora unet_full+te_full ...]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402

LEGS = ("unet_lora", "unet_lora+te_lora", "unet_lora+te_full", "unet_full", "unet_full+te_full")
ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=4)
ap.add_argument("--latent", type=int, default=64)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--legs", nargs="+", choices=LEGS, default=list(LEGS))
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_te.py measures on a GPU; none is visible")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def random_init(module):
    """Timing only: fan-in scaled random weights, embeddings N(0, 0.02), unit norm scales."""
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "embedding" in name and p.dim() == 2:
                p.normal_(0, 0.02)
            elif p.dim() > 1:
                p.normal_(0, p[0].numel() ** -0.5)
            elif "norm" in name and name.endswith("weight"):
                p.fill_(1.0)
            else:
                p.zero_()


def build(module):
    with torch.device("meta"):
        m = module()
    m = m.to_empty(device="cuda")
    random_init(m)
    return m.requires_grad_(False).eval()


def prompts(B, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((B, 77), 49407, dtype=torch.int64)
    ids[:, 0] = 49406
    for b in range(B):
        n = int(torch.randint(5, 70, (1,), generator=g))
        ids[b, 1:1 + n] = torch.randint(0, 49406, (n,), generator=g)
    return ids


def run_leg(leg):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    unet_part, _, te_part = leg.partition("+")
    unet = build(UNet2DConditionModel)
    if unet_part == "unet_full":
        groups, _ = make_hcpdiff(unet, [{"lr": 1e-6, "layers": [""]}], None)
    else:
        groups, _ = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 8, "layers": [r"re:.*\.attn.?$", r"re:.*\.ff$"]}])
    te, te_params = None, 0
    if te_part:
        te = build(CLIPTextModel)
        full, lora = ([{"lr": 1e-6, "layers": [""]}], None) if te_part == "te_full" else \
            (None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}])
        te_groups, _ = make_hcpdiff(te, full, lora, default_lr=1e-5)
        groups += te_groups
        te_params = sum(p.numel() for g in te_groups for p in g["params"])
    groups = [g for g in groups if len(g["params"])]
    step = LoraTrainStep(unet, groups, text_encoder=te, text_encoder_opts={"clip_skip": 0, "clip_final_norm": True} if te else None)
    B, S = args.batch, args.latent
    g = torch.Generator().manual_seed(0)
    lat, noise = torch.randn((B, 4, S, S), generator=g), torch.randn((B, 4, S, S), generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    ehs = prompts(B) if te is not None else torch.randn((B, 77, 768), generator=g)
    batch = [x.pin_memory() for x in (lat, noise, t, ehs)]
    for _ in range(max(args.warmup, 1)):
        step.step(*batch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step.step(*batch)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    out = {"ms_per_step": round(ms, 3), "images_per_s": round(B / ms * 1e3, 2),
           "trained_params": sum(p.numel() for g in groups for p in g["params"]), "te_trained_params": te_params,
           "optimizer_state_bytes": step.optimizer_state_bytes, "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "launches_per_step": step.launches_per_step, "loss": float(step.loss.cpu())}
    del step, unet, te, groups
    return out


result = {"workload": f"SD1.5 UNet + CLIP-L text encoder, AdamW, bs={args.batch}, {args.latent * 8}x{args.latent * 8}, 77 tokens",
          "gpu": card(), "steps": args.steps, "warmup": args.warmup}
for leg in args.legs:
    result[leg] = run_leg(leg)
print(json.dumps(result), flush=True)
