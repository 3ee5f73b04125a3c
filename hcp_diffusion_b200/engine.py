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

import torch
import torch.distributed as dist
from torch import nn

from . import _lib, ops
from ._lib import call, stream_ptr

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
    """One optimisation step of LoRA (or full) training on a `UNet2DConditionModel`: eps-prediction loss, grad-norm clip, AdamW.

    `params`: parameters, or optimizer-style groups [{'params': [...], 'lr': ..., 'weight_decay': ...}] (one per `lora_unet:` /
    `unet:` config item, reference cfg_net_tools.py:96-127).  `grad_accum_steps`: micro-batches per optimizer step
    (`train.gradient_accumulation_steps`).  `loss`: None / 'mse' or {'type': 'min_snr' | 'soft_min_snr' | 'kdiff_min_snr' | 'edm',
    'gamma': g}.  `ema`: None or {'decay_max', 'inv_gamma', 'power'} (ModelEMA defaults).  `cfg_scale`: None or the reference's
    `train.cfg_scale` string / (lo, hi, fn) for DreamArtist training: the UNet then runs on the doubled batch
    [latents | latents] against a text embedding of 2B rows [negative | positive]."""

    def __init__(self, unet: nn.Module, params: Union[Iterable[nn.Parameter], Sequence[dict]], lr: float = 1e-4, betas=(0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 1e-2, max_grad_norm: float = 1.0, use_cuda_graph: bool = True,
                 process_group: Optional[dist.ProcessGroup] = None, side_stream: bool = True, grad_accum_steps: int = 1,
                 loss: Union[None, str, dict] = None, ema: Optional[dict] = None, cfg_scale=None, num_train_timesteps: int = 1000):
        self.unet = unet
        params = list(params)
        if params and isinstance(params[0], dict):
            groups = [{"params": list(g["params"]), "lr": float(g.get("lr", lr)), "weight_decay": float(g.get("weight_decay", weight_decay))}
                      for g in params if len(list(g["params"]))]
        else:
            groups = [{"params": params, "lr": float(lr), "weight_decay": float(weight_decay)}]
        seen, flat_list = set(), []
        for g in groups:                                   # a parameter belongs to the first group that names it (torch.optim raises)
            g["params"] = [p for p in dict.fromkeys(g["params"]) if id(p) not in seen]
            seen.update(id(p) for p in g["params"])
            flat_list += g["params"]
        self.flat = FlatParams(flat_list)
        dev = self.flat.data.device
        self.m = torch.zeros_like(self.flat.data)
        self.v = torch.zeros_like(self.flat.data)
        # parameter groups = contiguous segments of the flat buffer, each with a device-side lr and step counter
        self.segments, i0 = [], 0
        for g in groups:
            n = len(g["params"])
            if n == 0:
                continue
            lo, hi = self.flat.offsets[i0], self.flat.end_of(i0 + n - 1)
            hyper = torch.tensor([g["lr"], betas[0], betas[1], eps, g["weight_decay"]], dtype=torch.float32, device=dev)
            self.segments.append({"lo": lo, "hi": hi, "hyper": hyper, "lr": hyper[0:1], "base_lr": g["lr"],
                                  "step": torch.zeros(1, dtype=torch.int32, device=dev)})
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
        self.acp = ddpm_alphas_cumprod(num_train_timesteps).to(dev)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
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

    def set_lr(self, lr: float, group: Optional[int] = None):
        """Set the lr of one group, or scale every group's configured lr by lr / base lr of group 0 (what an LR scheduler does)."""
        if group is not None:
            self.segments[group]["lr"].fill_(lr)
            return
        ratio = lr / self.segments[0]["base_lr"] if self.segments[0]["base_lr"] else 0.0
        for s in self.segments:
            s["lr"].fill_(s["base_lr"] * ratio)

    def set_hyper(self, group: int, lr: Optional[float] = None, beta1: Optional[float] = None):
        """What an LR scheduler writes per step (OneCycleLR cycles the lr and, for Adam, beta1): device-side, graph-replay safe."""
        h = self.segments[group]["hyper"]
        if lr is not None:
            h[0:1].fill_(lr)
        if beta1 is not None:
            h[1:2].fill_(beta1)

    def sync_params(self, src: int = 0):
        """DDP's construction-time broadcast (reference: accelerate `prepare` -> DistributedDataParallel): every replica starts
        from rank `src`'s trainable parameters."""
        if self.world > 1:
            dist.broadcast(self.flat.data, src=src, group=self.pg)
            if self.ema is not None:
                self.ema.copy_(self.flat.data)

    # ---- pieces ------------------------------------------------------------------------------------------------------
    def _forward_backward(self, latents, noise, t, ehs, added=None):
        """x_t = add_noise, pred = unet(x_t, t, ehs), loss, backward (gradients ACCUMULATE into the flat buffer)."""
        self.loss.zero_()
        ops.set_side_stream(self.side_stream)
        overlap = self.buckets is not None and self._micro == self.accum - 1      # DDP no_sync on all but the last micro-step
        if overlap:
            ops.set_grad_ready_callback(self.buckets.on_grad)
        try:
            self._fb_body(latents, noise, t, ehs, added)
        finally:
            ops.set_grad_ready_callback(None)
            ops.join_side()
            ops.set_side_stream(False)
        ops.advance_dropout()

    def _fb_body(self, latents, noise, t, ehs, added=None):
        B = latents.shape[0]
        per_image = latents[0].numel()
        x_t = torch.empty_like(latents)
        call("hcp_add_noise", latents.data_ptr(), noise.data_ptr(), t.data_ptr(), self.acp.data_ptr(), B, per_image, x_t.data_ptr(),
             stream_ptr())
        x_in, t_in = x_t, t
        if self.cfg_ctx is not None:                       # DreamArtistPTContext.pre: 'b c h w -> (pn b) c h w', timesteps.repeat(2)
            x_in, t_in = torch.cat([x_t, x_t], 0), torch.cat([t, t], 0)
        pred = (self.unet(x_in, t_in, ehs, added_cond_kwargs=added) if added is not None else self.unet(x_in, t_in, ehs)).sample
        if self.cfg_ctx is not None:
            pred = _CfgMixFn.apply(pred, t, *self.cfg_ctx)
        leaf = pred.detach()
        self.noise_pred = leaf
        dpred = torch.empty_like(leaf)
        gscale = 1.0 / self.accum                          # accelerator.backward: loss / gradient_accumulation_steps
        if self.loss_cfg is None:
            call("hcp_mse_loss", leaf.data_ptr(), noise.data_ptr(), leaf.numel(), gscale, self.loss.data_ptr(), dpred.data_ptr(), stream_ptr())
        else:
            mode, gamma = self.loss_cfg
            call("hcp_snr_mse_loss", leaf.data_ptr(), noise.data_ptr(), t.data_ptr(), self.acp.data_ptr(), gamma, mode, per_image, leaf.numel(),
                 gscale, self.loss.data_ptr(), dpred.data_ptr(), stream_ptr())
        pred.backward(dpred)

    def _optimizer(self):
        self.gsq.zero_()
        n = self.flat.numel
        call("hcp_sumsq", self.flat.grad.data_ptr(), n, self.gsq.data_ptr(), stream_ptr())
        for s in self.segments:
            lo, cnt = s["lo"], s["hi"] - s["lo"]
            call("hcp_adamw_flat_dev", self.flat.data.data_ptr() + 4 * lo, self.flat.grad.data_ptr() + 4 * lo, self.m.data_ptr() + 4 * lo,
                 self.v.data_ptr() + 4 * lo, cnt, s["hyper"].data_ptr(), 1.0 / self.world, self.gsq.data_ptr(), float(self.max_norm or 0.0),
                 s["step"].data_ptr(), stream_ptr())
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
        `cfg_scale`) (host-pinned or device); `added_cond_kwargs` ({'text_embeds' [B,P], 'time_ids' [B,6]}) for SDXL UNets
        (reference wrapper.py:66).  The optimizer runs on every `grad_accum_steps`-th call.  Returns the device loss tensor
        (shape [1]) of this micro-batch; reading it is the caller's D2H."""
        dev = self.flat.data.device
        if not self.use_graph:
            added = None if added_cond_kwargs is None else {k: v.to(dev, non_blocking=True) for k, v in added_cond_kwargs.items()}
            self._forward_backward(latents.to(dev, non_blocking=True), noise.to(dev, non_blocking=True), t.to(dev, non_blocking=True),
                                   ehs.to(dev, non_blocking=True), added)
            self._finish_micro(self._optimizer)
            return self.loss
        if self._static is None:
            self._capture(latents, noise, t, ehs, added_cond_kwargs)
        s = self._static
        s["latents"].copy_(latents, non_blocking=True)
        s["noise"].copy_(noise, non_blocking=True)
        s["t"].copy_(t, non_blocking=True)
        s["ehs"].copy_(ehs, non_blocking=True)
        if s["added"] is not None:
            for k, v in s["added"].items():
                v.copy_(added_cond_kwargs[k], non_blocking=True)
        self._graph_fb.replay()
        self._finish_micro(self._graph_opt.replay)
        return self.loss

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
        return (self.flat.data.clone(), self.m.clone(), self.v.clone(), [s["step"].clone() for s in self.segments],
                None if self.ema is None else self.ema.clone(), ops.dropout_state_snapshot())

    def _restore(self, saved):
        self.flat.data.copy_(saved[0]); self.m.copy_(saved[1]); self.v.copy_(saved[2])
        for s, c in zip(self.segments, saved[3]):
            s["step"].copy_(c)
        if self.ema is not None:
            self.ema.copy_(saved[4])
        ops.dropout_state_restore(saved[5])
        self.flat.grad.zero_()

    def _capture(self, latents, noise, t, ehs, added=None):
        dev = self.flat.data.device
        self._static = {
            "latents": latents.to(dev).float().contiguous().clone(), "noise": noise.to(dev).float().contiguous().clone(),
            "t": t.to(dev).long().contiguous().clone(), "ehs": ehs.to(dev).float().contiguous().clone(),
            "added": None if added is None else {k: v.to(dev).float().contiguous().clone() for k, v in added.items()},
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
                self._forward_backward(s["latents"], s["noise"], s["t"], s["ehs"], s["added"])
                self._optimizer()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._restore(saved)
        before = _lib.launch_count
        self._graph_fb = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph_fb):
            self._forward_backward(s["latents"], s["noise"], s["t"], s["ehs"], s["added"])
        self._graph_opt = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph_opt):
            self._optimizer()
        self.launches_per_step = _lib.launch_count - before
        # capture does not execute: nothing to restore, but the accumulated-gradient buffer must start clean
        self.flat.grad.zero_()


TrainStep = LoraTrainStep
