"""`python -m hcp_diffusion_b200.train_ac --cfg cfgs/train/lora_sd15_synthetic.yaml key=value ...`

The reference entrypoint (hcpdiff/train_ac.py:559-566: `load_config_with_cli` -> `Trainer(conf)` -> `trainer.train()`), reduced to
the hot path: build the UNet (cfg `model.unet`, the reference's injection seam train_ac.py:220), apply the `unet:` (full-layer
training) and `lora_unet:` lists through `make_hcpdiff` (train_ac.py:324-359), then run `train.train_steps` optimizer steps with
the H100 engine and save `ckpts/unet-<step>.safetensors` every `train.save_step` in the reference checkpoint format
(train_ac.py:523-544).  Honoured `train.*` keys: `gradient_accumulation_steps`, `max_grad_norm`, `scale_lr`, `optimizer.{lr,
weight_decay, betas, eps}`, `scheduler.{name, num_warmup_steps, num_training_steps, scheduler_kwargs}` (one_cycle / constant /
constant_with_warmup), `loss.criterion` (`torch.nn.MSELoss` or `hcpdiff.loss.MinSNRLoss`-family `_target_` + `gamma`), `cfg_scale`
(DreamArtist), `resume.{ckpt_path.unet, start_step}`; `model.ema` (`decay_max`, `inv_gamma`, `power`).

Out of the hot path and therefore NOT here: datasets / buckets / captions, the CLIP text encoder, VAE, loggers, DeepSpeed /
Colossal-AI trainers.  Inputs are the synthetic latents / text embeddings of SURVEY.md 8d (`data.synthetic`), or tensors saved
in a .pt file (`data.path`: {'latents': [N,4,h,w], 'encoder_hidden_states': [N,L,768]}).

Launch data-parallel with torchrun (one process per GPU); gradients are all-reduced over NCCL, every replica starts from rank
0's parameters (DDP's construction-time broadcast), the learning rate is scaled by batch x world x accumulation when
`train.scale_lr` is set (reference train_ac.py:192-197).
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

from .ckpt_manager import CkptManagerPKL, CkptManagerSafe, auto_manager
from .engine import LoraTrainStep
from .utils.cfg_net_tools import load_lora_state, make_hcpdiff
from .utils.config import instantiate, load_config_with_cli

_SNR_LOSSES = ("MinSNRLoss", "SoftMinSNRLoss", "KDiffMinSNRLoss", "EDMLoss")


def loss_from_cfg(loss_cfg):
    """`train.loss.criterion` -> engine loss spec.  `_target_: torch.nn.MSELoss` (train_base.yaml:26-29) -> None;
    `_target_: hcpdiff.loss.MinSNRLoss`, `gamma` (examples/min_snr.yaml) -> {'type', 'gamma'}."""
    crit = (loss_cfg or {}).get("criterion") if loss_cfg else None
    if not crit:
        return None
    if (loss_cfg.get("type", "eps") or "eps") != "eps":
        raise NotImplementedError("train.loss.type: only 'eps' (noise prediction) is on the hot path")
    target = str(crit.get("_target_", "torch.nn.MSELoss")).rsplit(".", 1)[-1]
    if target == "MSELoss":
        return None
    if target in _SNR_LOSSES:
        return {"type": target, "gamma": float(crit.get("gamma", 1.0))}
    raise NotImplementedError(f"train.loss.criterion {target!r} is not supported on the H100 hot path")


def make_scheduler(cfg, step_fn: LoraTrainStep):
    """Reference get_scheduler_with_name (hcpdiff/utils/net_utils.py:22-82) driven on a stand-in optimizer with the engine's groups:
    the real torch schedulers produce the numbers, `step()` copies lr (and OneCycleLR's cycled beta1) to the device."""
    if not cfg or not cfg.get("name"):
        return None
    name = cfg["name"]
    warm, total = int(cfg.get("num_warmup_steps", 0)), int(cfg.get("num_training_steps", 1))
    kwargs = dict(cfg.get("scheduler_kwargs") or {})
    dummy = [torch.nn.Parameter(torch.zeros(1)) for _ in step_fn.segments]
    opt = torch.optim.AdamW([{"params": [d], "lr": s["base_lr"]} for d, s in zip(dummy, step_fn.segments)], betas=tuple(step_fn.betas))
    if name == "one_cycle":
        sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=[s["base_lr"] for s in step_fn.segments], steps_per_epoch=total, epochs=1,
                                                    pct_start=warm / max(total, 1), **kwargs)
    elif name == "constant":
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda _: 1.0)
    elif name == "constant_with_warmup":
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, float(s) / float(max(1, warm))))
    else:
        raise NotImplementedError(f"train.scheduler.name={name!r}: one of one_cycle, constant, constant_with_warmup")

    def push():
        for i, g in enumerate(opt.param_groups):
            step_fn.set_hyper(i, lr=float(g["lr"]), beta1=float(g["betas"][0]))

    def step():
        opt.step()              # keeps torch's "optimizer.step() before lr_scheduler.step()" contract on the stand-in
        sched.step()
        push()

    push()
    return step


class Trainer:
    def __init__(self, cfgs):
        self.cfgs = cfgs
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local_rank)
        self.device = torch.device("cuda", self.local_rank)
        if self.world > 1 and not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            dist.init_process_group("nccl", device_id=self.device)
        seed = int(cfgs.get("seed", 114514))
        # The reference seeds with seed + local_rank (train_ac.py:128) and lets DDP broadcast rank 0's parameters at construction.
        # Here the model and the adapters are BUILT from the same seed on every rank (identical replicas without a 3.4 GB broadcast of
        # the frozen base) and only the data / noise / dropout streams are offset by the rank; trainable tensors are still broadcast.
        torch.manual_seed(seed)

        unet = cfgs.model.get("unet")
        unet = instantiate(unet) if isinstance(unet, dict) else unet
        if unet is None:
            raise ValueError("cfg `model.unet` must instantiate a UNet (e.g. _target_: hcp_diffusion_b200.models.UNet2DConditionModel)")
        init = cfgs.model.get("init")
        if init and init != "random":            # "random"/absent: keep the constructor's initialisation (no weights on disk here)
            sd = auto_manager(init).load_ckpt(init)
            unet.load_state_dict(sd.get("base", sd), strict=False)
        self.unet = unet.to(self.device).requires_grad_(False).eval()
        self.unet.enable_xformers_memory_efficient_attention()                      # no-ops kept for config compatibility
        if cfgs.model.get("gradient_checkpointing", False):
            self.unet.enable_gradient_checkpointing()

        tr = cfgs.train
        bs = int(cfgs.data.get("batch_size", 4))
        accum = int(tr.get("gradient_accumulation_steps", 1))
        lr_scale = bs * self.world * accum if tr.get("scale_lr", False) else 1
        opt_cfg = tr.get("optimizer") or {}
        groups, self.lora = make_hcpdiff(self.unet, cfgs.get("unet"), cfgs.get("lora_unet"), default_lr=float(opt_cfg.get("lr", 1e-4)))
        groups = [{"params": g["params"], "lr": float(g["lr"]) * lr_scale} for g in groups if len(g["params"])]
        resume = tr.get("resume")
        self.start_step = 0
        if resume:
            for path in (resume.get("ckpt_path", {}) or {}).get("unet", []) or []:
                sd = auto_manager(path).load_ckpt(path)
                if "base" in sd:
                    self.unet.load_state_dict(sd["base"], strict=False)
                if "lora" in sd:
                    load_lora_state(self.lora, sd["lora"])           # INTO the blocks being trained (see load_lora_state)
                    self.unet.load_state_dict(sd["lora"], strict=False)   # raw-key checkpoints (plugin_from_raw), as the reference does
            self.start_step = int(resume.get("start_step", 0) or 0)
        ema_cfg = cfgs.model.get("ema")
        ema = None
        if ema_cfg:
            ema = {k: ema_cfg[k] for k in ("decay_max", "inv_gamma", "power") if k in ema_cfg}
        cfg_scale = tr.get("cfg_scale")
        self.step_fn = LoraTrainStep(self.unet, groups, weight_decay=float(opt_cfg.get("weight_decay", 1e-2)),
                                     betas=tuple(opt_cfg.get("betas", (0.9, 0.999))), eps=float(opt_cfg.get("eps", 1e-8)),
                                     max_grad_norm=float(tr.get("max_grad_norm", 1.0)), use_cuda_graph=bool(tr.get("cuda_graph", True)),
                                     grad_accum_steps=accum, loss=loss_from_cfg(tr.get("loss")), ema=ema,
                                     cfg_scale=None if cfg_scale in (None, "1.0", 1.0) else str(cfg_scale))
        self.step_fn.sync_params(src=0)
        self.sched_step = make_scheduler(tr.get("scheduler"), self.step_fn)
        self.bs, self.accum = bs, accum
        self.cfg_doubled = self.step_fn.cfg_ctx is not None
        self.ckpt = CkptManagerSafe() if cfgs.get("ckpt_type", "safetensors") == "safetensors" else CkptManagerPKL()
        self.exp_dir = cfgs.get("exp_dir", "exps/run")
        if self.rank == 0:
            self.ckpt.set_save_dir(os.path.join(self.exp_dir, "ckpts"))
        from . import ops
        ops.set_dropout_seed(seed + 7919 * (self.rank + 1))
        self._load_data(seed)

    def _load_data(self, seed: int):
        d = self.cfgs.data
        g = torch.Generator().manual_seed(1234 + self.rank)
        if d.get("path"):
            blob = torch.load(d.path, map_location="cpu")
            self.latents, self.ehs = blob["latents"].float(), blob["encoder_hidden_states"].float()
            self.ehs_neg = blob.get("negative_hidden_states")
        else:
            n = int(d.get("num_samples", 64))
            s = int(self.unet.config.sample_size)
            gd = torch.Generator().manual_seed(seed)             # the synthetic "dataset" is the same on every rank; the sampling differs
            self.latents = torch.randn((n, self.unet.config.in_channels, s, s), generator=gd)
            self.ehs = torch.randn((n, int(d.get("tokens", 77)), self.unet.config.cross_attention_dim), generator=gd)
            self.ehs_neg = torch.randn((n, int(d.get("tokens", 77)), self.unet.config.cross_attention_dim), generator=gd)
        self.gen = g

    def next_batch(self):
        idx = torch.randint(0, self.latents.shape[0], (self.bs,), generator=self.gen)
        lat, ehs = self.latents[idx], self.ehs[idx]
        if self.cfg_doubled:                                     # DreamArtist: text embeddings [negative | positive]
            neg = self.ehs_neg[idx] if self.ehs_neg is not None else torch.zeros_like(ehs)
            ehs = torch.cat([neg, ehs], 0)
        noise = torch.randn(lat.shape, generator=self.gen)
        t = torch.randint(0, 1000, (self.bs,), generator=self.gen, dtype=torch.int64)
        return [x.pin_memory() for x in (lat, noise, t, ehs)]

    def save(self, step: int):
        base_trained = any(p.requires_grad for n, p in self.unet.named_parameters() if "lora_block_" not in n)
        path = self.ckpt.save_model_with_lora(self.unet if base_trained else None, self.lora, "unet", step,
                                              ema_state=self.step_fn.ema_state() if self.step_fn.ema is not None else None)
        return path

    def train(self):
        tr = self.cfgs.train
        steps, save_step, log_step = int(tr.train_steps), int(tr.get("save_step", 0)), int(tr.get("log_step", 20))
        t0, seen = time.time(), 0
        for step in range(self.start_step + 1, steps + 1):
            for _ in range(self.accum):
                loss = self.step_fn.step(*self.next_batch())
            if self.sched_step is not None:
                self.sched_step()
            seen += self.bs * self.world * self.accum
            if step % log_step == 0 or step == steps:
                val = float(loss.cpu())
                if self.rank == 0:
                    print(f"step {step}/{steps}  loss {val:.5f}  {seen / (time.time() - t0):.1f} img/s", flush=True)
                t0, seen = time.time(), 0
            if save_step and step % save_step == 0 and self.rank == 0:
                self.save(step)
        if self.world > 1:
            dist.barrier()


def main(argv=None):
    ap = argparse.ArgumentParser(description="HCP-Diffusion LoRA training on the H100 hot path")
    ap.add_argument("--cfg", type=str, required=True)
    args, overrides = ap.parse_known_args(argv)
    conf = load_config_with_cli(args.cfg, args_list=overrides)
    Trainer(conf).train()


if __name__ == "__main__":
    main(sys.argv[1:])
