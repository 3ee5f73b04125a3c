"""The training step around the UNet call, H100-native.

What the reference does per step (hcpdiff/train_ac.py:467-504): H2D copies, `make_noise` (:437-447), the CFG context
(`DreamArtistPTContext.pre/post`, hcpdiff/models/cfg_context.py:12-38), UNet forward through accelerate's autocast + DDP, the
criterion in fp32 (:506-515; `nn.MSELoss` or the SNR-weighted losses of hcpdiff/loss/min_snr_loss.py), `accelerator.backward`
(loss / accumulation steps; DDP all-reduce of the gradients on the last micro-step of `accelerator.accumulate`),
`clip_grad_norm_` (:485-490), AdamW with one lr per config item, `zero_grad`, `update_ema` (hcpdiff/utils/ema.py:18-32), and a
`loss.item()` sync.

Here: every trainable tensor is a view into ONE flat fp32 buffer (same for gradients, Adam moments and the EMA copy), so
  * zero_grad is one memset, clip + AdamW (+ EMA) are a handful of kernels over the flat buffer (no host sync: the clip factor is
    computed on the device); parameter groups are contiguous segments of the buffer with their own device-side lr,
  * the data-parallel exchange is ONE NCCL all-reduce of the flat gradient (6.4 MB for rank-8 attention LoRA) over
    NVLink/NVSwitch on the last micro-step -- the only collective in the job, exactly as the reference's DDP,
  * forward + loss + backward is captured once in a CUDA graph and replayed (about 1.2k kernel launches per step); the optimizer
    side is a second graph.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence, Union

import numpy as np
import torch
import torch.distributed as dist
from torch import nn

from . import _lib, adafactor, adamw8bit, ops, prodigy
from ._lib import call, stream_ptr
from .models.clip import SDXLTextEncoder, encode_prompt, encode_prompt_sdxl
from .noise import resolve as resolve_noise_schedule

SNR_LOSS_MODES = {"min_snr": 0, "soft_min_snr": 1, "kdiff_min_snr": 2, "edm": 3,
                  "MinSNRLoss": 0, "SoftMinSNRLoss": 1, "KDiffMinSNRLoss": 2, "EDMLoss": 3}
CFG_RATE_MODES = {"ln": 0, "cos": 1, "cos2": 2}


def ddpm_alphas_cumprod(num_steps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012) -> torch.Tensor:
    """SD1.5 DDPMScheduler(beta_schedule='scaled_linear') alphas_cumprod (constants as in reference tools/gen_from_ptlist.py:14-16)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_steps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def get_cfg_range(cfg_text: str):
    """'3.0' -> (3, 3, 'ln');  '1.0-3.0:cos' -> (1, 3, 'cos')   (reference hcpdiff/utils/utils.py:74-84)."""
    text, fn = str(cfg_text), "ln"
    if ":" in text:
        text, fn = text.split(":")
    if "-" in text:
        lo, hi = text.split("-")
        return float(lo), float(hi), fn
    return float(text), float(text), fn


class FlatParams:
    """Re-homes a list of parameters into one contiguous fp32 buffer (+ gradient buffer); names/shapes are untouched, so
    state_dict(), the optimizer param groups and hcpdiff's checkpoint code keep working."""

    def __init__(self, params: Sequence[nn.Parameter]):
        params = [p for p in dict.fromkeys(params)]
        if not params:
            raise ValueError("no trainable parameters")
        dev = params[0].device
        self.params = params
        self.offsets, n = [], 0
        for p in params:
            if p.dtype != torch.float32:
                raise TypeError("trainable parameters must be fp32 master weights")
            self.offsets.append(n)
            n += (p.numel() + 3) // 4 * 4          # keep every tensor 16-byte aligned inside the flat buffer
        self.numel = n
        self.data = torch.zeros(n, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)
        for p, o in zip(params, self.offsets):
            view = self.data[o:o + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
            p.grad = self.grad[o:o + p.numel()].view_as(p)

    def zero_grad(self):
        self.grad.zero_()

    def end_of(self, i: int) -> int:
        return self.offsets[i + 1] if i + 1 < len(self.offsets) else self.numel


class GradBuckets:
    """Bucketed all-reduce of the flat gradient buffer, overlapped with the backward pass (the reference: DistributedDataParallel's
    reducer, 25 MB buckets launched from autograd hooks).  The flat buffer is cut into contiguous ranges of about `bucket_bytes`; the
    weight-gradient kernels report the parameters they have just produced (ops.notify_grad), and when the last parameter of a range
    has been reported the range is all-reduced over NCCL on a communication stream ordered after the producing kernels.  The
    optimizer waits for the communication stream.  Parameters nobody reported (frozen / unused) are flushed by `finish()`."""

    def __init__(self, flat: FlatParams, pg, bucket_bytes: int = 256 << 20):
        self.flat, self.pg = flat, pg
        self.comm = torch.cuda.Stream()
        per = max(bucket_bytes // 4, 1)
        self.ranges, self.bucket_of = [], {}
        lo, k = 0, 0
        for i, p in enumerate(flat.params):
            self.bucket_of[id(p)] = k
            hi = flat.end_of(i)
            if hi - lo >= per or i == len(flat.params) - 1:
                self.ranges.append((lo, hi))
                lo, k = hi, k + 1
        self.count = [0] * len(self.ranges)
        for p in flat.params:
            self.count[self.bucket_of[id(p)]] += 1
        self.reset()

    def reset(self):
        self.remaining = list(self.count)
        self.seen = set()
        self.launched = [False] * len(self.ranges)

    def on_grad(self, params):
        for p in params:
            k = self.bucket_of.get(id(p))
            if k is None or id(p) in self.seen:
                continue
            self.seen.add(id(p))
            self.remaining[k] -= 1
            if self.remaining[k] == 0:
                self._launch(k)

    def _launch(self, k):
        if self.launched[k]:
            return
        self.launched[k] = True
        lo, hi = self.ranges[k]
        ev = torch.cuda.Event()
        ev.record()                                       # after the kernels that produced the bucket's last gradient
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(ev)
            dist.all_reduce(self.flat.grad[lo:hi], op=dist.ReduceOp.SUM, group=self.pg)

    def finish(self):
        for k in range(len(self.ranges)):
            self._launch(k)
        torch.cuda.current_stream().wait_stream(self.comm)
        self.reset()


class _CfgMixFn(torch.autograd.Function):
    """DreamArtistPTContext.post (cfg_context.py:23-39) on the doubled-batch prediction [uncond | cond]."""

    @staticmethod
    def forward(ctx, eps2: torch.Tensor, t: torch.Tensor, lo: float, hi: float, mode: int, T: int):
        eps2 = eps2.float().contiguous()
        B = eps2.shape[0] // 2
        out = torch.empty((B, *eps2.shape[1:]), dtype=torch.float32, device=eps2.device)
        call("hcp_cfg_mix_f32", eps2.data_ptr(), None, t.data_ptr(), B, eps2[0].numel(), lo, hi, mode, T, out.data_ptr(), stream_ptr())
        ctx.save_for_backward(t)
        ctx.cfg = (lo, hi, mode, T, B)
        return out

    @staticmethod
    def backward(ctx, dout):
        (t,) = ctx.saved_tensors
        lo, hi, mode, T, B = ctx.cfg
        dout = dout.float().contiguous()
        d2 = torch.empty((2 * B, *dout.shape[1:]), dtype=torch.float32, device=dout.device)
        call("hcp_cfg_mix_f32", None, dout.data_ptr(), t.data_ptr(), B, dout[0].numel(), lo, hi, mode, T, d2.data_ptr(), stream_ptr())
        return d2, None, None, None, None, None


class LoraTrainStep:
    """One optimisation step of LoRA (or full) training on a `UNet2DConditionModel`: eps-prediction loss, grad-norm clip, AdamW
    (or Adafactor, Lion, AdamW8bit or Prodigy).

    `params`: parameters, or optimizer-style groups [{'params': [...], 'lr': ..., 'weight_decay': ...}] (one per `lora_unet:` /
    `unet:` config item, reference cfg_net_tools.py:96-127).  `grad_accum_steps`: micro-batches per optimizer step
    (`train.gradient_accumulation_steps`).  `loss`: None / 'mse' or {'type': 'min_snr' | 'soft_min_snr' | 'kdiff_min_snr' | 'edm',
    'gamma': g}.  `ema`: None or {'decay_max', 'inv_gamma', 'power'} (ModelEMA defaults).  `cfg_scale`: None or the reference's
    `train.cfg_scale` string / (lo, hi, fn) for DreamArtist training: the UNet then runs on the doubled batch
    [latents | latents] against a text embedding of 2B rows [negative | positive].

    `optimizer`: 'adamw' (torch.optim.AdamW with `lr`, `betas`, `eps`, `weight_decay`; betas / weight_decay default to
    (0.9, 0.999) / 1e-2), 'lion' (lion_pytorch.Lion with `lr`, `betas`, `weight_decay`, defaults (0.9, 0.99) / 0.0: one flat
    momentum buffer, half of AdamW's state) or 'adafactor' (transformers.optimization.Adafactor; `optimizer_kwargs` takes its
    constructor keys with its defaults -- `lr`, `eps`, `clip_threshold`, `decay_rate`, `beta1`, `weight_decay`, `scale_parameter`,
    `relative_step`, `warmup_init` -- and a group's own 'lr' / 'weight_decay' win over them).  Adafactor keeps factored second moments per tensor of the module's shape (state sized by
    adafactor.state_numel), plus one flat first-moment buffer only when `beta1` is set.  'adamw8bit' is bitsandbytes.optim.AdamW8bit
    (`lr`, `betas`, `eps`, `weight_decay` with AdamW's defaults; `optimizer_kwargs` takes its constructor keys -- those four win
    over the arguments when given, and `min_8bit_size`, default 4096 -- and refuses the options adamw8bit.check_options refuses):
    tensors of at least min_8bit_size elements keep both moments as 8-bit codes with one fp32 scale per 256-element block (about
    2 B per parameter), smaller ones fp32 moments; weight decay is applied after the step, as bitsandbytes applies it.  'prodigy'
    is prodigyopt.Prodigy (`lr`, `betas`, `eps`, `weight_decay` with its defaults 1.0, (0.9, 0.999), 1e-8, 0.0; `optimizer_kwargs`
    takes `beta3`, `d0`, `d_coef`, `growth_rate`, `use_bias_correction`, `safeguard_warmup`, `decouple`): p0, s, m, v per
    parameter (16 B) and the step size d estimated on the device; every group's lr must be the largest lr or 0, as prodigyopt
    requires.

    `text_encoder`: a `models.CLIPTextModel` whose LoRA adapters (the reference's `lora_text_encoder`) and / or base parameters
    (`text_encoder:`, full fine-tuning) train together with the UNet (`TEUnetWrapper`); every trainable text-encoder parameter must be
    among `params` (their own groups), so they share the flat buffer: one all-reduce, one global-norm clip over both models, the same
    optimizer and EMA.  The token table [vocab, C] is one tensor of the flat buffer like any other: the rows no prompt used get a
    zero gradient, and every optimizer treats them as it treats any zero gradient (AdamW / Lion / AdamW8bit / Prodigy still move
    them by their moments and weight decay, Adafactor's factored second moment spans the whole table), as torch.optim does with
    a dense nn.Embedding gradient.  `step()` then takes int64 token ids [B, 77 R] in place of the
    text embedding, and the text encoder runs forward and backward inside the same graph.  `text_encoder_opts`: {'n_repeats',
    'clip_skip', 'clip_final_norm'} of `models.encode_prompt`.  With an SDXL (text_time) UNet the text encoder is a
    `models.SDXLTextEncoder` (SDXLTEUnetWrapper): `step()` takes ids [B, 2 x 77] and `added_cond_kwargs={'time_ids'}`, and
    `text_embeds` is the encoder's projected pooled row (`models.encode_prompt_sdxl`; n_repeats 1).

    `loss_weights`: one weight per data group of `step_groups()` (the reference's per-dataset `loss_weight`, e.g. DreamBooth's
    prior-preservation class set); None weighs every group 1.0.

    `noise_scheduler`: None (SD1.x's scaled_linear DDPM table over `num_train_timesteps`, default 1000), the reference's
    `model.noise_scheduler` config or a resolved `noise.NoiseSchedule`.  Its alphas_cumprod table serves add_noise, the Min-SNR
    weights and the grouped loss, and its T the CFG rate (a different `num_train_timesteps` is an error).  With a
    PyramidNoiseScheduler the base N(0,1) noise the caller passes becomes pyramid noise on the device, per data group and
    micro-step (`ops.PyramidNoise`; seed it with `set_noise_seed`), and the loss target is the un-normalised pyramid sum, as in the
    reference."""

    def __init__(self, unet: nn.Module, params: Union[Iterable[nn.Parameter], Sequence[dict]], lr: Optional[float] = None, betas=None,
                 eps: float = 1e-8, weight_decay: Optional[float] = None, max_grad_norm: float = 1.0, use_cuda_graph: bool = True,
                 process_group: Optional[dist.ProcessGroup] = None, side_stream: bool = True, grad_accum_steps: int = 1,
                 loss: Union[None, str, dict] = None, ema: Optional[dict] = None, cfg_scale=None,
                 optimizer: str = "adamw", optimizer_kwargs: Optional[dict] = None, text_encoder: Optional[nn.Module] = None,
                 text_encoder_opts: Optional[dict] = None, loss_weights: Optional[Sequence[float]] = None,
                 noise_scheduler=None, num_train_timesteps: Optional[int] = None):
        self.unet = unet
        self.loss_weights = None if loss_weights is None else [float(w) for w in loss_weights]
        self._group_tables: Dict[tuple, dict] = {}
        self.te, self.te_opts, self.sdxl = text_encoder, None, False
        if text_encoder is not None:
            if cfg_scale is not None:
                raise NotImplementedError("cfg_scale (DreamArtist batch doubling) together with a trained text encoder is not supported")
            opts = dict(text_encoder_opts or {})
            unknown = set(opts) - {"n_repeats", "clip_skip", "clip_final_norm"}
            if unknown:
                raise ValueError(f"text_encoder_opts: unknown keys {sorted(unknown)}")
            self.te_opts = {"n_repeats": int(opts.get("n_repeats", 1)), "clip_skip": int(opts.get("clip_skip", 0)),
                            "clip_final_norm": bool(opts.get("clip_final_norm", True))}
            self.sdxl = getattr(getattr(unet, "config", None), "addition_embed_type", None) == "text_time"
            if self.sdxl != isinstance(text_encoder, SDXLTextEncoder):
                raise NotImplementedError("an SDXL (text_time) UNet trains with an SDXLTextEncoder (its pooled bigG projection is "
                                          "text_embeds), and an SDXLTextEncoder needs an SDXL UNet")
            if self.sdxl and self.te_opts["n_repeats"] != 1:
                raise NotImplementedError(
                    "SDXL with n_repeats > 1 (tokenizer_repeats) is not supported: the reference pools bigG's text_embeds at the "
                    "largest id of the raw tokenizer output before it is cut into 77-token chunks, which pre-chunked ids cannot "
                    "express (the reference's SDXL config uses tokenizer_repeats: 1)")
        if optimizer not in ("adamw", "adafactor", "lion", "adamw8bit", "prodigy"):
            raise ValueError(f"optimizer {optimizer!r}: one of 'adamw', 'adafactor', 'lion', 'adamw8bit', 'prodigy'")
        self.optimizer = optimizer
        default_betas, default_wd = {"lion": ((0.9, 0.99), 0.0), "prodigy": ((0.9, 0.999), 0.0)}.get(optimizer, ((0.9, 0.999), 1e-2))
        betas = default_betas if betas is None else tuple(betas)
        weight_decay = default_wd if weight_decay is None else weight_decay
        lr = (1.0 if optimizer == "prodigy" else 1e-4) if lr is None else lr
        af_opts = a8_opts = pd_opts = None
        if optimizer == "prodigy":
            pd_opts = prodigy.engine_options(optimizer_kwargs)
        elif optimizer == "adamw8bit":
            given = dict(optimizer_kwargs or {})
            a8_opts = adamw8bit.check_options(given)
            lr = a8_opts["lr"] if "lr" in given else lr
            betas = a8_opts["betas"] if "betas" in given else betas
            eps = a8_opts["eps"] if "eps" in given else eps
            weight_decay = a8_opts["weight_decay"] if "weight_decay" in given else weight_decay
        elif optimizer == "adafactor":
            af_opts = adafactor.check_options(optimizer_kwargs)
            weight_decay = af_opts["weight_decay"]
            if af_opts["lr"] is not None:
                lr = af_opts["lr"]
        elif optimizer_kwargs:
            raise ValueError("optimizer_kwargs are the Adafactor options; AdamW and Lion take lr / betas / weight_decay (AdamW also eps)")
        params = list(params)
        if params and isinstance(params[0], dict):
            groups = [{"params": list(g["params"]), "lr": float(g.get("lr", lr)), "weight_decay": float(g.get("weight_decay", weight_decay))}
                      for g in params if len(list(g["params"]))]
        else:
            groups = [{"params": params, "lr": float(lr), "weight_decay": float(weight_decay)}]
        if pd_opts is not None:
            prodigy.check_lrs([g["lr"] for g in groups])
        seen, flat_list = set(), []
        for g in groups:                                   # a parameter belongs to the first group that names it (torch.optim raises)
            g["params"] = [p for p in dict.fromkeys(g["params"]) if id(p) not in seen]
            seen.update(id(p) for p in g["params"])
            flat_list += g["params"]
        if text_encoder is not None:
            missing = [n for n, p in text_encoder.named_parameters() if p.requires_grad and id(p) not in seen]
            if missing:
                raise ValueError(f"text-encoder parameters {missing[:3]}... are trainable but not in `params`: pass the "
                                 "text_encoder / lora_text_encoder groups too (they share the flat buffer, the clip and the optimizer)")
        self.flat = FlatParams(flat_list)
        dev = self.flat.data.device
        self.m = self.v = None
        if af_opts is not None:
            self._init_adafactor(groups, af_opts)
        elif a8_opts is not None:
            self._init_adamw8bit(groups, a8_opts, betas, eps)
        elif pd_opts is not None:
            self._init_prodigy(groups, pd_opts, betas, eps)
        else:
            self.m = torch.zeros_like(self.flat.data)
            self.v = torch.zeros_like(self.flat.data) if optimizer == "adamw" else None
        # parameter groups = contiguous segments of the flat buffer, each with a device-side lr and step counter
        self.segments, i0 = [], 0
        for g in groups:
            n = len(g["params"])
            if n == 0:
                continue
            lo, hi = self.flat.offsets[i0], self.flat.end_of(i0 + n - 1)
            if af_opts is not None:                        # rows of the [groups, 8] table the Adafactor kernels read
                gi = len(self.segments)
                hyper, step = self.af_hyper[gi], self.af_steps[gi:gi + 1]
            elif a8_opts is not None:                      # rows of the [groups, 5] table the AdamW8bit kernel reads
                gi = len(self.segments)
                hyper, step = self.a8_hyper[gi], self.a8_steps[gi:gi + 1]
            elif pd_opts is not None:                      # {offset, count, lr, weight_decay} rows the Prodigy kernels read
                gi = len(self.segments)
                hyper, step = self.pd_segs_f64[gi, 2:], self.pd_step
            else:
                hyper = torch.tensor([g["lr"], betas[0], betas[1], eps, g["weight_decay"]], dtype=torch.float32, device=dev)
                step = torch.zeros(1, dtype=torch.int32, device=dev)
            self.segments.append({"lo": lo, "hi": hi, "hyper": hyper, "lr": hyper[0:1], "base_lr": g["lr"], "step": step})
            i0 += n
        self.lr = self.segments[0]["lr"]
        self.step_count = self.segments[0]["step"]
        self.betas, self.eps, self.max_norm = betas, eps, max_grad_norm
        self.accum = max(int(grad_accum_steps), 1)
        self._micro = 0
        if isinstance(loss, str):
            loss = None if loss in ("mse", "MSELoss") else {"type": loss}
        self.loss_cfg = None
        if loss is not None:
            kind = loss.get("type", "min_snr")
            if kind not in SNR_LOSS_MODES:
                raise ValueError(f"unknown loss {kind!r}: one of mse, {sorted(SNR_LOSS_MODES)}")
            self.loss_cfg = (SNR_LOSS_MODES[kind], float(loss.get("gamma", 1.0)))
        self.noise_sched = None if noise_scheduler is None else resolve_noise_schedule(noise_scheduler, loss)
        if self.noise_sched is not None:
            T = self.noise_sched.num_train_timesteps
            if num_train_timesteps is not None and int(num_train_timesteps) != T:
                raise ValueError(f"num_train_timesteps={num_train_timesteps} disagrees with the noise scheduler's {T}")
            num_train_timesteps = T
        num_train_timesteps = 1000 if num_train_timesteps is None else int(num_train_timesteps)
        self.cfg_ctx = None
        if cfg_scale is not None:
            lo, hi, fn = get_cfg_range(cfg_scale) if isinstance(cfg_scale, str) else cfg_scale
            if hi != 1.0:                                  # reference train_ac.py:83-86: scale 1.0 keeps the plain CFGContext
                if fn not in CFG_RATE_MODES:
                    raise NotImplementedError(f"cfg_scale rate function {fn!r}: one of {sorted(CFG_RATE_MODES)}")
                self.cfg_ctx = (float(lo), float(hi), CFG_RATE_MODES[fn], int(num_train_timesteps))
        self.ema_cfg, self.ema = None, None
        if ema is not None:
            self.ema_cfg = (float(ema.get("decay_max", 0.9997)), float(ema.get("inv_gamma", 1.0)), float(ema.get("power", 2 / 3)))
            self.ema = self.flat.data.clone()
        if self.noise_sched is None:
            self.acp = ddpm_alphas_cumprod(num_train_timesteps).to(dev)
        else:
            self.acp = self.noise_sched.alphas_cumprod.to(dev)
        pyr = None if self.noise_sched is None else self.noise_sched.pyramid
        self.pyramid = None if pyr is None else ops.PyramidNoise(pyr["level"], pyr["discount"], pyr["step_size"], dev)
        self.loss: Optional[torch.Tensor] = None           # the loss tensor of the last micro-step ([1] after step(), [G] after step_groups())
        self.noise_pred: Optional[torch.Tensor] = None     # the UNet output of the last micro-step (kept alive across graph replays)
        self.gsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.use_graph = use_cuda_graph
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self._static = None
        self._graph_fb = None
        self._graph_opt = None
        # data parallel + eager launches + a large gradient (full fine-tune: 3.4 GB): bucketed all-reduce overlapped with backward;
        # otherwise (LoRA: 6 MB; or CUDA graphs) one all-reduce between the two graphs
        self.buckets = None
        if self.world > 1 and not use_cuda_graph and self.flat.numel * 4 >= (64 << 20):
            self.buckets = GradBuckets(self.flat, process_group)
        # work off the critical path (LoRA-gradient kernels, text-embedding k/v projections) goes to a side stream inside
        # _forward_backward and is joined there, before anything reads the gradients (HCP_SIDE_STREAM=0 keeps a single stream)
        self.side_stream = side_stream

    def _init_adafactor(self, groups, opts):
        dev = self.flat.data.device
        groups = [g for g in groups if g["params"]]          # the segments: a group emptied by de-duplication has none
        group_of = [gi for gi, g in enumerate(groups) for _ in g["params"]]
        self.af_layout = adafactor.Layout([tuple(p.shape) for p in self.flat.params], self.flat.offsets, group_of)
        lay = self.af_layout
        rows = [adafactor.hyper_row(opts, g["lr"], g["weight_decay"]) for g in groups]
        self.af_hyper = torch.tensor(rows, dtype=torch.float32, device=dev)
        self.af_steps = torch.zeros(len(groups), dtype=torch.int32, device=dev)
        self.af_state = torch.zeros(lay.state_numel, dtype=torch.float32, device=dev)
        self.af_exp_avg = torch.zeros_like(self.flat.data) if opts["beta1"] is not None else None
        self.af_work = torch.zeros(lay.work_numel, dtype=torch.float32, device=dev)
        to_dev = lambda a: torch.from_numpy(a.view(np.uint8).copy()).to(dev)      # noqa: E731  (packed C structs)
        self.af_tensors, self.af_items = to_dev(lay.tensors), to_dev(lay.items)
        self.af_factor_items = to_dev(lay.factor_items) if lay.factor_items.size else None

    def _init_adamw8bit(self, groups, opts, betas, eps):
        dev = self.flat.data.device
        groups = [g for g in groups if g["params"]]          # the segments: a group emptied by de-duplication has none
        group_of = [gi for gi, g in enumerate(groups) for _ in g["params"]]
        self.a8_layout = lay = adamw8bit.Layout([p.numel() for p in self.flat.params], self.flat.offsets, group_of, opts["min_8bit_size"])
        self.a8_hyper = torch.tensor([[g["lr"], betas[0], betas[1], eps, g["weight_decay"]] for g in groups], dtype=torch.float32, device=dev)
        self.a8_steps = torch.zeros(len(groups), dtype=torch.int32, device=dev)
        self.a8_codes = torch.zeros(2 * lay.code_bytes, dtype=torch.uint8, device=dev)
        self.a8_absmax = torch.zeros(2 * lay.nblocks, dtype=torch.float32, device=dev)
        self.a8_state32 = torch.zeros(2 * lay.small_numel, dtype=torch.float32, device=dev)
        self.a8_maps = adamw8bit.maps().to(dev)
        to_dev = lambda a: torch.from_numpy(a.view(np.uint8).copy()).to(dev)      # noqa: E731  (packed C structs)
        self.a8_tensors, self.a8_items = to_dev(lay.tensors), to_dev(lay.items)

    def _init_prodigy(self, groups, opts, betas, eps):
        dev = self.flat.data.device
        groups = [g for g in groups if g["params"]]          # the segments: a group emptied by de-duplication has none
        rows, i0 = [], 0
        for g in groups:
            lo, hi = self.flat.offsets[i0], self.flat.end_of(i0 + len(g["params"]) - 1)
            rows.append((lo, hi - lo, g["lr"], g["weight_decay"]))
            i0 += len(g["params"])
        self.pd_segs_host = prodigy.segment_table(rows)
        self.pd_segs = torch.from_numpy(self.pd_segs_host.view(np.int64).reshape(len(rows), 4).copy()).to(dev)
        self.pd_segs_f64 = self.pd_segs.view(torch.float64)  # columns 2, 3: lr, weight_decay (set_lr / set_hyper write lr here)
        self.pd_hyper = torch.tensor(prodigy.hyper_row(opts, betas[0], betas[1], eps), dtype=torch.float64, device=dev)
        self.pd_state = torch.tensor(prodigy.initial_state(opts["d0"]), dtype=torch.float64, device=dev)
        self.pd_work = torch.zeros(prodigy.WORKSPACE_BYTES // 8, dtype=torch.float64, device=dev)
        self.pd_step = torch.zeros(1, dtype=torch.int32, device=dev)   # optimizer calls, skipped ones included (ModelEMA's step)
        self.pd_p0, self.pd_s = torch.zeros_like(self.flat.data), torch.zeros_like(self.flat.data)
        self.m, self.v = torch.zeros_like(self.flat.data), torch.zeros_like(self.flat.data)

    @property
    def optimizer_state_bytes(self) -> int:
        """Bytes of optimizer state (moments; not the parameters, gradients or scratch)."""
        if self.optimizer == "adamw8bit":
            return sum(b.numel() * b.element_size() for b in (self.a8_codes, self.a8_absmax, self.a8_state32))
        if self.optimizer == "adafactor":
            return 4 * (self.af_state.numel() + (0 if self.af_exp_avg is None else self.af_exp_avg.numel()))
        if self.optimizer == "prodigy":
            return 4 * sum(b.numel() for b in (self.pd_p0, self.pd_s, self.m, self.v))
        return 4 * sum(b.numel() for b in (self.m, self.v) if b is not None)

    def _opt_buffers(self) -> List[torch.Tensor]:
        if self.optimizer == "adamw8bit":
            return [self.a8_codes, self.a8_absmax, self.a8_state32, self.a8_steps]
        if self.optimizer == "prodigy":
            return [self.pd_p0, self.pd_s, self.m, self.v, self.pd_state, self.pd_step]
        if self.optimizer == "adafactor":
            return [self.af_state, self.af_steps] + ([] if self.af_exp_avg is None else [self.af_exp_avg])
        return [b for b in (self.m, self.v) if b is not None] + [s["step"] for s in self.segments]

    def set_lr(self, lr: float, group: Optional[int] = None):
        """Set the lr of one group, or scale every group's configured lr by lr / base lr of group 0 (what an LR scheduler does)."""
        if group is not None:
            self.segments[group]["lr"].fill_(lr)
            return
        ratio = lr / self.segments[0]["base_lr"] if self.segments[0]["base_lr"] else 0.0
        for s in self.segments:
            s["lr"].fill_(s["base_lr"] * ratio)

    def set_hyper(self, group: int, lr: Optional[float] = None, beta1: Optional[float] = None):
        """What an LR scheduler writes per step (OneCycleLR cycles the lr and, for AdamW, AdamW8bit, Lion and Prodigy, beta1):
        device-side, graph-replay safe.  Prodigy reads the betas of group 0 only, as prodigyopt does."""
        if self.optimizer == "prodigy":
            if lr is not None:
                self.segments[group]["lr"].fill_(lr)
            if beta1 is not None and group == 0:
                self.pd_hyper[0:1].fill_(beta1)
            return
        h = self.segments[group]["hyper"]
        if lr is not None:
            h[0:1].fill_(lr)
        if beta1 is not None:
            if self.optimizer == "adafactor":
                raise ValueError("beta1 is scheduled for AdamW, AdamW8bit and Lion only")
            h[1:2].fill_(beta1)

    def sync_params(self, src: int = 0):
        """DDP's construction-time broadcast (reference: accelerate `prepare` -> DistributedDataParallel): every replica starts
        from rank `src`'s trainable parameters."""
        if self.world > 1:
            dist.broadcast(self.flat.data, src=src, group=self.pg)
            if self.ema is not None:
                self.ema.copy_(self.flat.data)

    # ---- pieces ------------------------------------------------------------------------------------------------------
    def _forward_backward(self, latents, noise, t, ehs, added=None, tables=None, mask=None):
        """x_t = add_noise, pred = unet(x_t, t, ehs), loss, backward (gradients ACCUMULATE into the flat buffer).  `tables`: the
        device tables of the batch's group layout (`_tables`; None: one group of weight 1), `mask` fp32 [B, HW] or None; the
        per-group weighted, masked loss goes to tables['loss'], which becomes `self.loss`."""
        if tables is None:
            tables = self._tables((latents.shape[0],), (1.0,), latents.shape[1], latents[0, 0].numel())
        self.loss = tables["loss"]
        self.loss.zero_()
        ops.set_side_stream(self.side_stream)
        overlap = self.buckets is not None and self._micro == self.accum - 1      # DDP no_sync on all but the last micro-step
        if overlap:
            ops.set_grad_ready_callback(self.buckets.on_grad)
        try:
            self._fb_body(latents, noise, t, ehs, added, tables, mask)
        finally:
            ops.set_grad_ready_callback(None)
            ops.join_side()
            ops.set_side_stream(False)
        ops.advance_dropout()
        if self.pyramid is not None:
            self.pyramid.advance()

    def set_noise_seed(self, seed: int) -> None:
        """Seed of the pyramid noise draws (one per data-parallel rank, as the dropout seed); no-op without a pyramid."""
        if self.pyramid is not None:
            self.pyramid.set_seed(seed)

    def _fb_body(self, latents, noise, t, ehs, added, tables, mask):
        B, C = latents.shape[:2]
        HW = latents[0, 0].numel()
        if self.pyramid is not None:                       # PyramidNoiseScheduler.add_noise per group; the loss target is its sum
            x_t, noise = self.pyramid.add_noise(latents, noise, t, self.acp, tables["sizes"])
        else:
            x_t = torch.empty_like(latents)
            call("hcp_add_noise_scaled", latents.data_ptr(), noise.data_ptr(), t.data_ptr(), self.acp.data_ptr(), tables["inv_std"].data_ptr(),
                 tables["group_start"].data_ptr(), 1, B, C * HW, x_t.data_ptr(), stream_ptr())
        x_in, t_in = x_t, t
        if self.cfg_ctx is not None:                       # DreamArtistPTContext.pre: 'b c h w -> (pn b) c h w', timesteps.repeat(2)
            x_in, t_in = torch.cat([x_t, x_t], 0), torch.cat([t, t], 0)
        if self.sdxl:                                      # SDXLTEUnetWrapper.forward: text_embeds = bigG's projected pooled row
            ehs, text_embeds = encode_prompt_sdxl(self.te, ehs, self.te_opts["clip_skip"], self.te_opts["clip_final_norm"])
            added = {**added, "text_embeds": text_embeds}
        elif self.te is not None:                          # TEUnetWrapper.forward: ehs = TE(ids) with its adapters in the graph
            ehs = encode_prompt(self.te, ehs, **self.te_opts)
        pred = (self.unet(x_in, t_in, ehs, added_cond_kwargs=added) if added is not None else self.unet(x_in, t_in, ehs)).sample
        if self.cfg_ctx is not None:
            pred = _CfgMixFn.apply(pred, t, *self.cfg_ctx)
        leaf = pred.detach()
        self.noise_pred = leaf
        dpred = torch.empty_like(leaf)
        gscale = 1.0 / self.accum                          # accelerator.backward: loss / gradient_accumulation_steps
        mode, gamma = self.loss_cfg if self.loss_cfg is not None else (-1, 1.0)
        ws = tables["ws"]                                  # sum_g loss_weight_g * (criterion * mask).mean() over the groups' samples
        call("hcp_eps_loss_grouped", leaf.data_ptr(), noise.data_ptr(), t.data_ptr(), self.acp.data_ptr(), _lib.ptr(mask),
             tables["scale"].data_ptr(), tables["group"].data_ptr(), tables["loss"].numel(), mode, gamma, B, C, HW,
             gscale, tables["loss"].data_ptr(), dpred.data_ptr(), ws.data_ptr(), ws.numel() * 4, stream_ptr())
        pred.backward(dpred)

    def _optimizer(self):
        self.gsq.zero_()
        n = self.flat.numel
        call("hcp_sumsq", self.flat.grad.data_ptr(), n, self.gsq.data_ptr(), stream_ptr())
        if self.optimizer == "adafactor":
            lay = self.af_layout
            call("hcp_adafactor_flat", self.flat.data.data_ptr(), self.flat.grad.data_ptr(), self.af_state.data_ptr(),
                 _lib.ptr(self.af_exp_avg), self.af_work.data_ptr(), self.af_tensors.data_ptr(), self.af_items.data_ptr(), lay.items.size,
                 _lib.ptr(self.af_factor_items), lay.factor_items.size, self.af_hyper.data_ptr(), self.af_steps.data_ptr(),
                 len(self.segments), 1.0 / self.world, self.gsq.data_ptr(), float(self.max_norm or 0.0), stream_ptr())
        elif self.optimizer == "adamw8bit":
            lay = self.a8_layout
            nz = lambda t: t.data_ptr() if t.numel() else None      # noqa: E731  (a buffer no tensor uses is passed as NULL)
            call("hcp_adamw8bit_flat", self.flat.data.data_ptr(), self.flat.grad.data_ptr(), nz(self.a8_codes), nz(self.a8_absmax),
                 nz(self.a8_state32), self.a8_maps.data_ptr(), lay.tensors.ctypes.data, self.a8_tensors.data_ptr(), len(lay.tensors), lay.items.ctypes.data,
                 self.a8_items.data_ptr(), lay.items.size, n, lay.code_bytes, lay.nblocks, lay.small_numel, self.a8_hyper.data_ptr(),
                 self.a8_steps.data_ptr(), len(self.segments), 1.0 / self.world, self.gsq.data_ptr(), float(self.max_norm or 0.0),
                 stream_ptr())
        elif self.optimizer == "prodigy":
            call("hcp_prodigy_flat", self.flat.data.data_ptr(), self.flat.grad.data_ptr(), self.pd_p0.data_ptr(), self.pd_s.data_ptr(),
                 self.m.data_ptr(), self.v.data_ptr(), n, self.pd_segs_host.ctypes.data, self.pd_segs.data_ptr(), len(self.segments),
                 self.pd_hyper.data_ptr(), self.pd_state.data_ptr(), self.pd_work.data_ptr(), self.pd_work.numel() * 8, 1.0 / self.world,
                 self.gsq.data_ptr(), float(self.max_norm or 0.0), self.pd_step.data_ptr(), stream_ptr())
        for s in (self.segments if self.optimizer in ("adamw", "lion") else ()):
            lo, cnt = s["lo"], s["hi"] - s["lo"]
            p, g, m = (b.data_ptr() + 4 * lo for b in (self.flat.data, self.flat.grad, self.m))
            tail = (1.0 / self.world, self.gsq.data_ptr(), float(self.max_norm or 0.0), s["step"].data_ptr(), stream_ptr())
            if self.optimizer == "lion":
                call("hcp_lion_flat_dev", p, g, m, cnt, s["hyper"].data_ptr(), *tail)
            else:
                call("hcp_adamw_flat_dev", p, g, m, self.v.data_ptr() + 4 * lo, cnt, s["hyper"].data_ptr(), *tail)
        if self.ema is not None:
            call("hcp_ema_flat", self.ema.data_ptr(), self.flat.data.data_ptr(), n, self.step_count.data_ptr(), *self.ema_cfg, stream_ptr())
        self.flat.grad.zero_()                             # optimizer.zero_grad() (reference train_ac.py:494)

    def _all_reduce(self):
        if self.world > 1:
            if self.buckets is not None:
                self.buckets.finish()                      # buckets were launched from the backward pass; flush the rest and join
            else:
                dist.all_reduce(self.flat.grad, op=dist.ReduceOp.SUM, group=self.pg)   # averaged by grad_scale = 1/world in AdamW

    def _finish_micro(self, run_opt):
        self._micro += 1
        if self._micro >= self.accum:                      # accelerator.sync_gradients
            self._micro = 0
            self._all_reduce()
            run_opt()

    # ---- public ------------------------------------------------------------------------------------------------------
    def step(self, latents: torch.Tensor, noise: torch.Tensor, t: torch.Tensor, ehs: torch.Tensor,
             added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
        """One micro-step: latents/noise fp32 [B,4,H,W], t int64 [B], ehs fp32 [B,L,ctx] ([2B,L,ctx] = [negative | positive] with
        `cfg_scale`), or int64 token ids [B, 77 R] with a `text_encoder` (host-pinned or device); `added_cond_kwargs` ({'text_embeds' [B,P], 'time_ids' [B,6]}) for SDXL UNets
        (reference wrapper.py:66; {'time_ids'} only, with ids [B, 2 x 77], when an SDXLTextEncoder is trained).  The optimizer runs on every `grad_accum_steps`-th call.  Returns the device loss tensor
        (shape [1]) of this micro-batch; reading it is the caller's D2H.  This is `step_groups()` with one group of weight 1.0
        (`loss_weights` does not apply), and shares its CUDA graphs when that layout was captured."""
        batch = {"latents": latents, "noise": noise, "t": t, "ehs": ehs}
        if added_cond_kwargs is not None:
            batch["added_cond_kwargs"] = added_cond_kwargs
        return self._run([batch], (1.0,))

    def step_groups(self, batches: Sequence[Dict[str, torch.Tensor]]) -> torch.Tensor:
        """One micro-step over several data groups (the reference's `cfgs.data` datasets, e.g. DreamBooth's instance set next to its
        prior-preservation class set; hcpdiff/train_ac.py:467-482).  `batches`: one dict per group, {'latents', 'noise', 't', 'ehs'}
        as `step()` takes them, plus optional 'added_cond_kwargs' and 'mask' (fp32 [B_g, h, w] or [B_g, 1, h, w] at latent
        resolution, the reference's att_mask weights; absent = ones).  The groups run as ONE UNet pass over their concatenation
        (every op is per-sample independent), and the loss is sum_g loss_weight_g * mean(criterion * mask) with each group's own
        mean, so the gradient is the reference's sum over per-group backward passes.  Groups share the latent shape, the text
        width and the added-cond layout.  Returns the device tensor fp32 [G] of the weighted per-group losses of this micro-step
        (the reference logs the last one)."""
        weights = self.loss_weights if self.loss_weights is not None else [1.0] * len(batches)
        if not batches or len(weights) != len(batches):
            raise ValueError(f"step_groups: {len(batches)} batches for {len(weights)} loss_weights")
        return self._run(batches, weights)

    def _run(self, batches, weights) -> torch.Tensor:
        """The micro-step of `step()` and `step_groups()`.  With CUDA graphs the first call captures them for its layout (group batch
        sizes, loss weights, mask or not); every later call of that layout copies its inputs into the captured buffers and replays."""
        lat, noise, t, ehs, added, mask, sizes = self._concat_groups(batches)
        layout = (sizes, tuple(weights), mask is not None)
        if self._static is not None and layout != self._static["layout"]:
            raise ValueError(f"the CUDA graphs were captured for the layout {self._static['layout']} (group batch sizes, loss weights, "
                             f"mask); this call's is {layout}: use one LoraTrainStep per layout")
        C, HW = lat.shape[1], lat[0, 0].numel()
        if not self.use_graph:
            dev = self.flat.data.device
            to_dev = lambda x: None if x is None else x.to(dev, non_blocking=True).contiguous()      # noqa: E731
            self._forward_backward(to_dev(lat), to_dev(noise), to_dev(t), to_dev(ehs),
                                   None if added is None else {k: to_dev(v) for k, v in added.items()},
                                   self._tables(sizes, weights, C, HW), to_dev(mask))
            self._finish_micro(self._optimizer)
            return self.loss
        if self._static is None:
            self._capture(lat, noise, t, ehs, added, self._tables(sizes, weights, C, HW), mask, layout)
        s = self._static
        for k, x in (("latents", lat), ("noise", noise), ("t", t), ("ehs", ehs), ("mask", mask)):
            if x is not None:
                s[k].copy_(x, non_blocking=True)
        if s["added"] is not None:
            for k, v in s["added"].items():
                v.copy_(added[k], non_blocking=True)
        return self.step_resident()

    def _concat_groups(self, batches):
        """Concatenate the groups' tensors along the batch in the layouts the step expects; refuse groups that cannot share a pass.
        One group's tensors are handed through as they are: torch.cat of one pinned host tensor returns pageable memory, which
        would make the H2D copies synchronous."""
        allowed = {"latents", "noise", "t", "ehs", "added_cond_kwargs", "mask"}
        sizes, lats, noises, ts, ehss, addeds, masks = [], [], [], [], [], [], []
        for g, b in enumerate(batches):
            unknown = set(b) - allowed
            if unknown:
                raise ValueError(f"group {g} has unknown keys {sorted(unknown)} (allowed: {sorted(allowed)})")
            lat, nz, tt, eh = b["latents"], b["noise"], b["t"], b["ehs"]
            B = lat.shape[0]
            if lat.dim() != 4 or tuple(nz.shape) != tuple(lat.shape) or tuple(tt.shape) != (B,):
                raise ValueError(f"group {g}: latents [B,C,h,w], noise of the same shape and t [B] (got "
                                 f"{tuple(lat.shape)}, {tuple(nz.shape)}, {tuple(tt.shape)})")
            if lats and tuple(lat.shape[1:]) != tuple(lats[0].shape[1:]):
                raise ValueError(f"group {g} latents {tuple(lat.shape[1:])} differ from group 0's "
                                 f"{tuple(lats[0].shape[1:])}: groups share one latent shape (buckets are not supported)")
            rows = 2 * B if self.cfg_ctx is not None else B
            if eh.shape[0] != rows:
                raise ValueError(f"group {g}: ehs has {eh.shape[0]} rows, expected {rows}"
                                 + (" ([negative | positive] with cfg_scale)" if self.cfg_ctx is not None else ""))
            if ehss and tuple(eh.shape[1:]) != tuple(ehss[0].shape[1:]):
                raise ValueError(f"group {g} ehs {tuple(eh.shape[1:])} differs from group 0's {tuple(ehss[0].shape[1:])}")
            ad = b.get("added_cond_kwargs")
            if self.sdxl:
                if not ad or "time_ids" not in ad:
                    raise ValueError(f"group {g}: an SDXL UNet with a text encoder needs added_cond_kwargs={{'time_ids': [B, 6]}}")
                if "text_embeds" in ad:
                    raise ValueError(f"group {g}: text_embeds is computed by the trained SDXL text encoder (bigG's projected pooled "
                                     "row): pass added_cond_kwargs={'time_ids'} only")
            if addeds and (ad is None) != (addeds[0] is None):
                raise ValueError(f"group {g}: added_cond_kwargs must be given for every group or for none")
            if ad is not None:
                if any(v.shape[0] != B for v in ad.values()):
                    raise ValueError(f"group {g}: added_cond_kwargs rows differ from its batch {B}")
                if addeds and ({k: tuple(v.shape[1:]) for k, v in ad.items()} != {k: tuple(v.shape[1:]) for k, v in addeds[0].items()}):
                    raise ValueError(f"group {g}: added_cond_kwargs layout differs from group 0's")
            m = b.get("mask")
            if m is not None:
                if tuple(m.shape) not in ((B,) + tuple(lat.shape[2:]), (B, 1) + tuple(lat.shape[2:])):
                    raise ValueError(f"group {g}: mask {tuple(m.shape)}, expected [{B}, h, w] or [{B}, 1, h, w] at latent "
                                     f"resolution {tuple(lat.shape[2:])}")
                m = m.reshape(B, -1).float()
            sizes.append(B)
            lats.append(lat), noises.append(nz), ts.append(tt), ehss.append(eh), addeds.append(ad), masks.append(m)
        cat = (lambda xs: xs[0]) if len(sizes) == 1 else (lambda xs: torch.cat(xs, 0))      # noqa: E731
        if self.cfg_ctx is not None and len(sizes) > 1:    # [neg_1 .. neg_G | pos_1 .. pos_G], the layout _CfgMixFn expects
            ehs = torch.cat([e[:B] for e, B in zip(ehss, sizes)] + [e[B:] for e, B in zip(ehss, sizes)], 0)
        else:
            ehs = cat(ehss)
        added = None if addeds[0] is None else {k: cat([a[k] for a in addeds]) for k in addeds[0]}
        mask = None
        if any(m is not None for m in masks):
            HW = lats[0][0, 0].numel()
            mask = cat([m if m is not None else torch.ones((B, HW), dtype=torch.float32, device=lats[g].device)
                        for g, (m, B) in enumerate(zip(masks, sizes))])
        return (cat(lats), cat(noises), cat(ts), ehs, added, mask, tuple(sizes))

    def _tables(self, sizes, weights, C, HW):
        """Device tables of one group layout (built once per layout): its sizes, sample_scale fp32 [B] = w_g / (B_g C HW),
        sample_group int32 [B], the per-group loss fp32 [G], the loss kernel's workspace, and the inv_std / group_start tables of
        add_noise without a pyramid: every 1/std is 1, so one group spans the batch whatever G is."""
        key = (sizes, tuple(weights), C, HW)
        tab = self._group_tables.get(key)
        if tab is None:
            dev = self.flat.data.device
            scale = [w / (B * C * HW) for w, B in zip(weights, sizes) for _ in range(B)]
            group = [g for g, B in enumerate(sizes) for _ in range(B)]
            nbytes = _lib.lib().hcp_eps_loss_grouped_workspace_bytes(sum(sizes), C * HW)
            tab = {"sizes": sizes, "scale": torch.tensor(scale, dtype=torch.float32, device=dev),
                   "group": torch.tensor(group, dtype=torch.int32, device=dev), "loss": torch.zeros(len(sizes), dtype=torch.float32, device=dev),
                   "ws": torch.zeros((nbytes + 3) // 4, dtype=torch.float32, device=dev),
                   "inv_std": torch.ones(1, dtype=torch.float32, device=dev),
                   "group_start": torch.tensor([0, sum(sizes)], dtype=torch.int32, device=dev)}
            self._group_tables[key] = tab
        return tab

    def step_resident(self) -> torch.Tensor:
        """Replay on the inputs already resident in the static device buffers (kernel-only timing in bench.py)."""
        if self._static is None:
            raise RuntimeError("call step() once before step_resident()")
        self._graph_fb.replay()
        self._finish_micro(self._graph_opt.replay)
        return self.loss

    def ema_state(self) -> Dict[nn.Parameter, torch.Tensor]:
        """{parameter: EMA tensor view} (what ModelEMA.state_dict() holds for the trainable parameters)."""
        if self.ema is None:
            return {}
        return {p: self.ema[o:o + p.numel()].view_as(p) for p, o in zip(self.flat.params, self.flat.offsets)}

    def _snapshot(self):
        return (self.flat.data.clone(), [b.clone() for b in self._opt_buffers()],
                None if self.ema is None else self.ema.clone(), ops.dropout_state_snapshot(),
                None if self.pyramid is None else self.pyramid.state.clone())

    def _restore(self, saved):
        self.flat.data.copy_(saved[0])
        for b, c in zip(self._opt_buffers(), saved[1]):
            b.copy_(c)
        if self.ema is not None:
            self.ema.copy_(saved[2])
        ops.dropout_state_restore(saved[3])
        if self.pyramid is not None:
            self.pyramid.state.copy_(saved[4])
        self.flat.grad.zero_()

    def _capture(self, latents, noise, t, ehs, added, tables, mask, layout):
        dev = self.flat.data.device
        self._static = {
            "latents": latents.to(dev).float().contiguous().clone(), "noise": noise.to(dev).float().contiguous().clone(),
            "t": t.to(dev).long().contiguous().clone(),
            "ehs": (ehs.to(dev).long() if self.te is not None else ehs.to(dev).float()).contiguous().clone(),
            "added": None if added is None else {k: v.to(dev).float().contiguous().clone() for k, v in added.items()},
            "mask": None if mask is None else mask.to(dev).float().contiguous().clone(),
            "tables": tables, "layout": layout,
        }
        s = self._static
        # warm-up on a side stream (builds the packed weights, tensor maps, autograd metadata) -- parameters, optimizer state and
        # the gradients accumulated so far (none: capture happens on the first micro-step) are restored
        if self._micro != 0:
            raise RuntimeError("CUDA-graph capture must happen on the first micro-step of an accumulation window")
        saved = self._snapshot()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._forward_backward(s["latents"], s["noise"], s["t"], s["ehs"], s["added"], s["tables"], s["mask"])
                self._optimizer()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._restore(saved)
        before = _lib.launch_count
        self._graph_fb = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph_fb):
            self._forward_backward(s["latents"], s["noise"], s["t"], s["ehs"], s["added"], s["tables"], s["mask"])
        self._graph_opt = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph_opt):
            self._optimizer()
        self.launches_per_step = _lib.launch_count - before
        # capture does not execute: nothing to restore, but the accumulated-gradient buffer must start clean
        self.flat.grad.zero_()


TrainStep = LoraTrainStep
