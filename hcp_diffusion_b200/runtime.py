"""Execution-side glue between the nn.Module tree (the plugin surface) and the packed kernel operands.

A `LinearGroup` owns the bf16 operands of one GEMM made of one or several sibling linear layers reading the same input
(to_q/to_k/to_v of a self-attention; to_k/to_v of a cross-attention; a single layer), each of which may be a plain
nn.Linear / 1x1 nn.Conv2d or a `LoraPatchContainer` carrying any number of stacked `LoraBlock`s.  Packs are rebuilt when the
module identities, the stacked plugins or the (in-place) version of a base weight change.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn

from . import _lib, ops
from .models.lora import DAPPPatchContainer, LoraBlock, LoraPatchContainer
from .ops import BF16, ConvLoraRef, ConvPack, LinearPack, LoraBlockRef


def host_and_blocks(child: nn.Module) -> Tuple[nn.Module, List[LoraBlock]]:
    """(base layer, [LoraBlock, ...]) of a linear-like child; anything else fails loudly (no silent eager fallback)."""
    if isinstance(child, LoraPatchContainer):
        blocks = [child[name] for name in child.plugin_names]
        for b in blocks:
            if not isinstance(b, LoraBlock):
                raise NotImplementedError(f"plugin {type(b).__name__} on a hot-path layer is not supported")
        return child._host, blocks
    if isinstance(child, (nn.Linear, nn.Conv2d)):
        return child, []
    raise NotImplementedError(f"layer type {type(child).__name__} on the UNet hot path is not supported by hcp_diffusion_b200")


def dropout_p(blocks: Sequence[LoraBlock]) -> float:
    """nn.Dropout probability applied to the patched layer's output: the reference container calls `self[name].post_forward` with
    the LAST plugin name of its loop (lora_base_patch.py:35,74; lora_layers_patch.py:128-131), i.e. the last block's dropout."""
    if not blocks:
        return 0.0
    d = blocks[-1].dropout
    return float(d.p) if (d.training and d.p > 0) else 0.0


def _versions(host: nn.Module, blocks: Sequence[LoraBlock]):
    """In-place edits that must invalidate a pack: base weight / bias, each block's alpha buffer, the dropout setting."""
    bias = getattr(host, "bias", None)
    return (host.weight._version, host.weight.data_ptr(), None if bias is None else (bias._version, bias.data_ptr()),
            tuple((id(b), b.alpha._version, getattr(b, "branch", None)) for b in blocks), dropout_p(blocks))


def _weight_2d(host: nn.Module) -> torch.Tensor:
    w = host.weight
    if isinstance(host, nn.Conv2d):
        if host.kernel_size != (1, 1):
            raise NotImplementedError("only 1x1 convolutions can be run as a linear group")
        return w.reshape(w.shape[0], w.shape[1])
    return w


class LinearGroup:
    def __init__(self, children: Sequence[nn.Module]):
        self.children = list(children)
        self.pack: Optional[LinearPack] = None
        self._sig = None
        self._k_splits = None
        self.drops = None

    def _signature(self, k_splits):
        sig = [tuple(k_splits) if k_splits else None, ops.LORA_MERGE, ops.WEIGHT_TILED, ops.LORA_EXT]
        for ch in self.children:
            host, blocks = host_and_blocks(ch)
            sig.append((id(ch), id(host), _versions(host, blocks)))
        return tuple(sig)

    def prepare(self, k_splits: Optional[Sequence[int]] = None) -> LinearPack:
        k_splits = k_splits or self._k_splits
        sig = self._signature(k_splits)
        if self.pack is not None and sig == self._sig:
            return self.pack
        hosts = [host_and_blocks(ch) for ch in self.children]
        for host, _ in hosts:
            if not host.weight.is_cuda:
                raise _lib.HcpError("hcp_diffusion_b200 runs on CUDA only: move the model to an H100 device (there is no CPU path)")
        w = torch.cat([_weight_2d(h) for h, _ in hosts], dim=0)
        biases = [h.bias for h, _ in hosts]
        bias = None
        if any(b is not None for b in biases):
            bias = torch.cat([b if b is not None else torch.zeros(h.weight.shape[0], device=w.device) for (h, _), b in zip(hosts, biases)])
        pack = LinearPack(w, bias, k_splits)
        o0 = 0
        for host, _ in hosts:                                    # full fine-tune (`unet:` config items): trained base layers
            n = host.weight.shape[0]
            if host.weight.requires_grad or (host.bias is not None and host.bias.requires_grad):
                if not host.weight.requires_grad:
                    raise NotImplementedError("training a bias without its weight is not supported")
                pack.train.append((host.weight, host.bias, o0, n))
            o0 += n
        refs, o0 = [], 0
        for ch, (host, blocks) in zip(self.children, hosts):
            dapp = isinstance(ch, DAPPPatchContainer)
            for b in blocks:
                branch = getattr(b, "branch", None) if dapp else None      # a plain LoraPatchContainer sums every block (ref. :21-35)
                if dapp and branch not in ("p", "n"):
                    continue                                               # DAPPPatchContainer.forward only reads 'p' / 'n' blocks
                refs.append(LoraBlockRef(b.layer.W_down, b.layer.W_up, float(b.alpha), o0, branch))
            o0 += host.weight.shape[0]
        if refs:
            pack.attach_lora(refs)
            if ops.LORA_MERGE:
                per_host, o0 = [], 0
                for host, _ in hosts:
                    n = host.weight.shape[0]
                    per_host.append((_weight_2d(host).detach(), o0, n, [r for r in refs if o0 <= r.o0 < o0 + n]))
                    o0 += n
                pack.enable_merge(per_host)
        if ops.WEIGHT_TILED:
            pack.tile_weights()
        # nn.Dropout of the patched children: column ranges of the fused output, None when nothing is dropped
        ranges, c0 = [], 0
        for host, blocks in hosts:
            ranges.append((c0, host.weight.shape[0], dropout_p(blocks)))
            c0 += host.weight.shape[0]
        self.drops = ranges if any(p > 0 for _, _, p in ranges) else None
        self.pack, self._sig, self._k_splits = pack, sig, k_splits
        return pack

    def __call__(self, xs: Sequence[torch.Tensor], residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        pack = self.prepare([x.shape[-1] for x in xs] if len(xs) > 1 else None)
        if self.drops is None:
            return ops.fused_linear(pack, xs, residual)
        # y = dropout(layer(x)) + residual: the residual leaves the GEMM epilogue and rides the dropout kernel instead
        return ops.dropout_cols(ops.fused_linear(pack, xs, None), self.drops, residual=residual)

    def run_standalone(self, x: torch.Tensor) -> torch.Tensor:
        """Used by LoraPatchContainer.forward: any float dtype in, same dtype out.  Linear hosts take [..., in]; 1x1 Conv2d hosts
        take NCHW like the reference layer (the NHWC view is the boundary conversion, the product path inside the UNet never
        leaves NHWC)."""
        if not x.is_cuda:
            raise _lib.HcpError("hcp_diffusion_b200 has no CPU path: LoRA layers run on an H100 only")
        pack = self.prepare()
        if pack.lora:
            pack_lora([self])
        host, _ = host_and_blocks(self.children[0])
        if isinstance(host, nn.Conv2d):
            B, C_, H, W = x.shape
            t = x.permute(0, 2, 3, 1).reshape(B, H * W, C_).to(BF16).contiguous()
            y = self([t])
            return y.view(B, H, W, -1).permute(0, 3, 1, 2).to(x.dtype)
        y = self([x.to(BF16)])
        return y.to(x.dtype)


class _JobTable:
    def __init__(self):
        self.key = None
        self.dev = self.cdev = self.mdev = self.mmap = None
        self.mrank = 0
        self.n = self.cn = self.mn = self.mtiles = 0


_job_table = _JobTable()


def pack_lora(groups: Sequence, table: Optional[_JobTable] = None) -> None:
    """One kernel launch that refreshes the packed low-rank operands of every LoRA-carrying group (LinearGroup / ConvGroup) from
    the fp32 parameters, plus one for the 3x3 down-projections of Conv2d LoRA blocks."""
    table = table or _JobTable()
    jobs, cjobs, mjobs = [], [], []
    for g in groups:
        if g.pack is not None and g.pack.lora:
            jobs += g.pack.jobs()
            if isinstance(g.pack, ConvPack):
                cjobs += g.pack.conv_jobs()
            elif g.pack.merged:
                mjobs += g.pack.merge_jobs()
    if not jobs:
        return
    key = (tuple((j.w_down, j.w_up, j.A, j.BlT, j.alpha) for j in jobs) + tuple((j.w_down, j.wt) for j in cjobs)
           + tuple((j.w_host, j.W, j.o0, j.nblocks, tuple(j.w_down), tuple(j.alpha)) for j in mjobs))
    if table.key != key:
        table.mdev, table.mn, table.mtiles, table.mmap = None, 0, 0, None
        if mjobs:
            tiles, tmap = 0, []
            for i, j in enumerate(mjobs):
                j.tile0 = tiles
                n = ((j.out_dim + 63) // 64) * ((j.in_dim + 63) // 64)
                tmap += [i] * n
                tiles += n
            table.mmap = torch.tensor(tmap, dtype=torch.int32).cuda()
            table.mrank = max(sum(j.rank[i] for i in range(j.nblocks)) for j in mjobs)
            marr = (_lib.LoraMergeJob * len(mjobs))(*mjobs)
            table.mdev = torch.frombuffer(bytearray(bytes(marr)), dtype=torch.uint8).cuda()
            table.mn, table.mtiles = len(mjobs), tiles
        arr = (_lib.LoraJob * len(jobs))(*jobs)
        table.dev = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
        table.cdev = None
        if cjobs:
            carr = (_lib.LoraConvJob * len(cjobs))(*cjobs)
            table.cdev = torch.frombuffer(bytearray(bytes(carr)), dtype=torch.uint8).cuda()
        table.key, table.n, table.cn = key, len(jobs), len(cjobs)
    _lib.call("hcp_lora_pack", table.dev.data_ptr(), table.n, _lib.stream_ptr())
    if table.mdev is not None:
        _lib.call("hcp_lora_merge", table.mdev.data_ptr(), table.mn, table.mtiles, table.mmap.data_ptr(), table.mrank, _lib.stream_ptr())
    if table.cdev is not None:
        _lib.call("hcp_lora_pack_conv", table.cdev.data_ptr(), table.cn, _lib.stream_ptr())


def repack_trained(groups: Sequence, table: Optional[_JobTable] = None, extra_jobs: Sequence = ()) -> None:
    """Full fine-tune: ONE launch refreshes the bf16 operands (W, W^T / the two 3x3 arrangements, fused biases) of every trained layer
    from the fp32 master parameters the optimizer just updated (the reference's autocast re-casts the fp32 weights every forward)."""
    jobs = list(extra_jobs)
    for g in groups:
        if g.pack is not None:
            jobs += g.pack.repack_jobs()
    if not jobs:
        return
    table = table or _JobTable()
    key = tuple((j.src, j.dst0, j.dst1, j.kind, j.o0) for j in jobs)
    if table.key != key:
        arr = (_lib.RepackJob * len(jobs))(*jobs)
        table.dev = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
        table.key, table.n = key, len(jobs)
    _lib.call("hcp_repack_weights", table.dev.data_ptr(), table.n, _lib.stream_ptr())


class ConvGroup:
    """Packed operands of one 3x3 convolution layer: a frozen nn.Conv2d, or a LoraPatchContainer around one (LoCon: LoraLayer
    blocks with W_down [r,Cin,3,3] / W_up [Cout,r,1,1], reference lora_layers_patch.py:64-100)."""

    def __init__(self, conv: nn.Module):
        self.conv = conv
        self.pack: Optional[ConvPack] = None
        self._sig = None
        self.drop_p = 0.0

    def prepare(self) -> ConvPack:
        child = self.conv
        dapp = isinstance(child, DAPPPatchContainer)
        conv, blocks = host_and_blocks(child)
        if not isinstance(conv, nn.Conv2d):
            raise NotImplementedError(f"{type(conv).__name__} on a 3x3 convolution of the hot path is not supported")
        sig = (id(child), id(conv), _versions(conv, blocks), ops.WEIGHT_TILED)
        if self.pack is None or sig != self._sig:
            if not conv.weight.is_cuda:
                raise _lib.HcpError("hcp_diffusion_b200 runs on CUDA only (there is no CPU path)")
            if conv.kernel_size != (3, 3) or conv.padding != (1, 1) or conv.stride[0] not in (1, 2):
                raise NotImplementedError("only 3x3 / pad 1 / stride 1|2 convolutions are supported")
            pack = ConvPack(conv.weight, conv.bias, conv.stride[0])
            if conv.weight.requires_grad:                        # full fine-tune
                pack.train = (conv.weight, conv.bias)
            refs = []
            for b in blocks:
                branch = getattr(b, "branch", None) if dapp else None
                if dapp and branch not in ("p", "n"):
                    continue                       # DAPPPatchContainer.forward only reads 'p' / 'n' blocks (lora_layers_patch.py:108-126)
                refs.append(ConvLoraRef(b.layer.W_down, b.layer.W_up, float(b.alpha), branch))
            if refs:
                pack.attach_lora(refs)
            if ops.WEIGHT_TILED:
                pack.tile_weights()
            self.drop_p = dropout_p(blocks)
            self.pack, self._sig = pack, sig
        return self.pack

    def __call__(self, x: torch.Tensor, geom, rowbias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """conv(x) [+ per-image row bias] [+ residual]; with nn.Dropout on the patched layer (reference lora_base_patch.py:74) the
        two additions leave the convolution epilogue and ride the dropout kernel: dropout(conv(x) + b) + rowbias + residual."""
        pack = self.prepare()
        if self.drop_p <= 0:
            return ops.conv3x3(pack, x, geom, rowbias=rowbias, residual=residual)
        y = ops.conv3x3(pack, x, geom)
        B, H, W = geom
        s = pack.stride
        return ops.dropout_cols(y, [(0, pack.Cout, self.drop_p)], residual=residual, rowbias=rowbias, rows_per_group=(H // s) * (W // s))

    def run_standalone(self, x: torch.Tensor) -> torch.Tensor:
        """LoraPatchContainer.forward on a 3x3 host: NCHW in / out like the reference layer."""
        if not x.is_cuda:
            raise _lib.HcpError("hcp_diffusion_b200 has no CPU path: LoRA layers run on an H100 only")
        pack = self.prepare()
        if pack.lora:
            pack_lora([self])
        B, C_, H, W = x.shape
        t = x.permute(0, 2, 3, 1).reshape(B, H * W, C_).to(BF16).contiguous()
        y = self(t, (B, H, W))
        s = pack.stride
        return y.view(B, H // s, W // s, -1).permute(0, 3, 1, 2).to(x.dtype)
