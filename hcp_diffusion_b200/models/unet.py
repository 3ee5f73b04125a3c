"""`UNet2DConditionModel` for the SD1.x topology, executed by the libhcpb200 kernels.

Drop-in for the model seam of the reference trainer: `unet = cfgs.model.get('unet') or UNet2DConditionModel.from_pretrained`
(hcpdiff/train_ac.py:220-222), called as `unet(noisy_latents, timesteps, encoder_hidden_states,
encoder_attention_mask=...).sample` (hcpdiff/models/wrapper.py:29).  The module tree reproduces the diffusers names and
parameter shapes pinned by the reference dump cfgs/unet_struct.txt (they are the public API: yaml `layers` regexes,
checkpoint keys, LoRA conversion), and every leaf is a real nn.Linear / nn.Conv2d / nn.GroupNorm / nn.LayerNorm that hcpdiff's
plugin surgery (delattr/setattr on the parent, hcpdiff/models/plugin.py:224-232) can replace.

Execution does not go through the leaves' own forward(): each block drives fused kernels over bf16 NHWC activations
(ops.py), keeping fp32 master parameters in the modules.  Boundary: NCHW fp32 (or any float) in, NCHW `sample.dtype` out.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn

from .. import _lib, ops
from ..runtime import ConvGroup, LinearGroup, _JobTable, pack_lora, repack_trained


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor


class Timesteps(nn.Module):
    """Parameter-free sinusoidal embedding (computed inside the time-embedding kernel)."""

    def __init__(self, num_channels: int):
        super().__init__()
        self.num_channels = num_channels


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)


class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, temb_channels: int, groups: int = 32, eps: float = 1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, stride=1, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, stride=1, padding=1)
        self.nonlinearity = nn.SiLU()
        if in_channels != out_channels:
            self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1, stride=1, padding=0)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.in_split = None              # (C_h, C_skip) when the block is fed the concatenation of two tensors (up blocks)
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(conv1=ConvGroup(self.conv1), conv2=ConvGroup(self.conv2),
                                shortcut=LinearGroup([self.conv_shortcut]) if hasattr(self, "conv_shortcut") else None)
            self.__dict__["_g"] = g
        # the children may have been swapped by plugin surgery since the last call
        g.conv1.conv, g.conv2.conv = self.conv1, self.conv2
        if g.shortcut is not None:
            g.shortcut.children = [self.conv_shortcut]
            if self.in_split is not None and g.shortcut._k_splits is None:
                g.shortcut._k_splits = list(self.in_split)     # known at construction: the packs are built once, before the first call
        return g

    def run(self, xs: Sequence[torch.Tensor], geom, temb: torch.Tensor) -> torch.Tensor:
        """xs: one tensor [B,HW,C] or (h, skip) to be concatenated along channels; temb fp32 [B, Cout] view."""
        g = self._groups()
        x2 = xs[1] if len(xs) == 2 else None
        n1 = self.norm1
        outs = ops.group_norm(n1.weight, n1.bias, n1.num_groups, n1.eps, True, xs[0], x2)
        y1, aliases = outs[0], outs[1:]
        h = g.conv1(y1, geom, rowbias=temb)
        n2 = self.norm2
        y2 = ops.group_norm(n2.weight, n2.bias, n2.num_groups, n2.eps, True, h, None)[0]
        if g.shortcut is not None:
            res = g.shortcut(list(aliases))
        else:
            res = aliases[0]
        return g.conv2(y2, geom, residual=res)


class Attention(nn.Module):
    """diffusers `Attention` (dumped as `CrossAttention` by older versions: cfgs/unet_struct.txt:17): to_q/to_k/to_v
    without bias, to_out = [Linear(bias), Dropout]."""

    def __init__(self, query_dim: int, cross_attention_dim: Optional[int], heads: int):
        super().__init__()
        kdim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.inner_dim = query_dim
        self.is_cross = cross_attention_dim is not None
        self.to_q = nn.Linear(query_dim, query_dim, bias=False)
        self.to_k = nn.Linear(kdim, query_dim, bias=False)
        self.to_v = nn.Linear(kdim, query_dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(query_dim, query_dim), nn.Dropout(0.0)])
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(qkv=LinearGroup([]), q=LinearGroup([]), kv=LinearGroup([]), out=LinearGroup([]))
            self.__dict__["_g"] = g
        g.qkv.children = [self.to_q, self.to_k, self.to_v]
        g.q.children = [self.to_q]
        g.kv.children = [self.to_k, self.to_v]
        g.out.children = [self.to_out[0]]
        return g

    def linear_groups(self) -> List[LinearGroup]:
        g = self._groups()
        return [g.kv, g.q, g.out] if self.is_cross else [g.qkv, g.out]

    def run(self, x: torch.Tensor, residual: torch.Tensor, context, kv_bias: Optional[torch.Tensor],
            kv: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`context`: the text embedding [B, Lc, ctx], a `_PerAttnContext` (one alias per cross-attention, when the embedding carries
        a gradient) or a `_HoistedKV` holding the k/v projections computed ahead of time; `kv`: those projections, already taken."""
        g = self._groups()
        C_ = self.inner_dim
        if not self.is_cross:
            qkv = g.qkv([x])                                                  # [B, L, 3C]: one GEMM, LoRA deltas block-diagonal
            o = ops.attention(self.heads, C_, (0, C_, 2 * C_), qkv, None, None)
        else:
            q = g.q([x])
            if kv is not None:
                pass
            elif isinstance(context, _HoistedKV):
                kv = context.take(self)
            else:
                kv = g.kv([context.take(self) if isinstance(context, _PerAttnContext) else context])   # [B, Lc, 2C]
            o = ops.attention(self.heads, C_, (0, 0, C_), q, kv, kv_bias)
        return g.out([o], residual=residual)


class _PerAttnContext:
    """The text embedding as one alias per cross-attention (ops.context_fanout): the k/v dgrads of the attentions come back as
    separate gradients and are summed in fp32 (the reference's per-use autocast casts of the fp32 embedding)."""

    def __init__(self, ehs: torch.Tensor, attns: Sequence["Attention"]):
        self.ctx = dict(zip((id(a) for a in attns), ops.context_fanout(ehs, len(attns))))

    def take(self, attn: "Attention") -> torch.Tensor:
        return self.ctx.pop(id(attn))


class _HoistedKV:
    """k/v projections of the text embedding for every cross-attention, issued on the side stream at the start of the forward
    (they depend on nothing but the text embedding, and autograd runs their backward -- incl. the LoRA-gradient kernels -- on
    the same side stream).  `take` makes the main stream wait for them once, at the first consumer."""

    def __init__(self, ctx, attns: Sequence["Attention"]):
        """`ctx`: the bf16 text embedding, or a `_PerAttnContext` when it carries a gradient."""
        self.ctx = ctx
        main = torch.cuda.current_stream()
        self.side = ops.fork_side(*(ctx.ctx.values() if isinstance(ctx, _PerAttnContext) else (ctx,)))
        self.joined = False
        self.kv = {}
        with torch.cuda.stream(self.side):
            for a in attns:
                t = a._groups().kv([ctx.take(a) if isinstance(ctx, _PerAttnContext) else ctx])
                t.record_stream(main)               # produced on the side stream, consumed (and later freed) on the main one
                self.kv[id(a)] = t

    def take(self, attn: "Attention") -> torch.Tensor:
        if not self.joined:
            torch.cuda.current_stream().wait_stream(self.side)
            self.joined = True
        return self.kv.pop(id(attn))


class GEGLU(nn.Module):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim: int, mult: int = 4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(proj=LinearGroup([]), out=LinearGroup([]))
            self.__dict__["_g"] = g
        g.proj.children = [self.net[0].proj]
        g.out.children = [self.net[2]]
        return g

    def linear_groups(self) -> List[LinearGroup]:
        g = self._groups()
        return [g.proj, g.out]

    def run(self, x: torch.Tensor, residual: torch.Tensor, skip_out: bool = False) -> torch.Tensor:
        """`skip_out`: the rerun of a recompute region, where the out-projection's forward GEMM is needed only when it also produces
        the merged-LoRA rank rows its backward reads."""
        g = self._groups()
        u = g.proj([x])
        h = ops.GegluFn.apply(u)
        if skip_out:
            with ops.skip_output():
                return g.out([h], residual=residual)
        return g.out([h], residual=residual)


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim: int, heads: int, cross_attention_dim: int, ln_eps: float = 1e-5):
        super().__init__()
        self.attn1 = Attention(dim, None, heads)
        self.ff = FeedForward(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads)
        self.norm1 = nn.LayerNorm(dim, eps=ln_eps)
        self.norm2 = nn.LayerNorm(dim, eps=ln_eps)
        self.norm3 = nn.LayerNorm(dim, eps=ln_eps)

    def run(self, h: torch.Tensor, context, kv_bias: Optional[torch.Tensor], checkpoint: bool = False) -> torch.Tensor:
        """`checkpoint`: run the block as one recompute region (ops.checkpoint).  The first pass keeps the block's input, the
        cross-attention's context (or its hoisted k/v) and each attention's output and LSE rows; the backward reruns the block from
        them.  The context enters the region as a tensor taken once, so the hoisted k/v projections are not recomputed."""
        if not checkpoint:
            return self._run(h, context, None, kv_bias)
        kv = context.take(self.attn2) if isinstance(context, _HoistedKV) else None
        c = kv if kv is not None else (context.take(self.attn2) if isinstance(context, _PerAttnContext) else context)
        params = [p for p in self.parameters() if p.requires_grad]
        if not (params or h.requires_grad or c.requires_grad):
            return self._run(h, c, kv, kv_bias)
        hoisted = kv is not None

        def region(h, c, recompute):
            return self._run(h, c, c if hoisted else None, kv_bias, recompute)
        return ops.checkpoint(region, (h, c), params)

    def _run(self, h, context, kv, kv_bias, recompute: bool = False) -> torch.Tensor:
        n, a = ops.layer_norm(self.norm1.weight, self.norm1.bias, self.norm1.eps, h)
        h = self.attn1.run(n, a, None, None)
        n, a = ops.layer_norm(self.norm2.weight, self.norm2.bias, self.norm2.eps, h)
        h = self.attn2.run(n, a, context, kv_bias, kv=kv)
        n, a = ops.layer_norm(self.norm3.weight, self.norm3.bias, self.norm3.eps, h)
        return self.ff.run(n, a, skip_out=recompute)


class Transformer2DModel(nn.Module):
    """GroupNorm -> proj_in -> `depth` BasicTransformerBlocks -> proj_out (+ residual).  proj_in / proj_out are 1x1 Conv2d (SD1.x)
    or nn.Linear (`use_linear_projection`, SDXL); on NHWC token matrices both are the same GEMM."""

    def __init__(self, channels: int, heads: int, cross_attention_dim: int, groups: int = 32, eps: float = 1e-6, depth: int = 1,
                 use_linear_projection: bool = False):
        super().__init__()
        self.norm = nn.GroupNorm(groups, channels, eps=eps, affine=True)
        self.proj_in = nn.Linear(channels, channels) if use_linear_projection else nn.Conv2d(channels, channels, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(channels, heads, cross_attention_dim) for _ in range(depth)])
        self.proj_out = nn.Linear(channels, channels) if use_linear_projection else nn.Conv2d(channels, channels, 1)
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(proj_in=LinearGroup([]), proj_out=LinearGroup([]))
            self.__dict__["_g"] = g
        g.proj_in.children = [self.proj_in]
        g.proj_out.children = [self.proj_out]
        return g

    def linear_groups(self) -> List[LinearGroup]:
        g = self._groups()
        return [g.proj_in, g.proj_out]

    def run(self, x: torch.Tensor, context: torch.Tensor, kv_bias: Optional[torch.Tensor], checkpoint: bool = False) -> torch.Tensor:
        g = self._groups()
        n = self.norm
        y, alias = ops.group_norm(n.weight, n.bias, n.num_groups, n.eps, False, x, None)
        h = g.proj_in([y])                      # NHWC tokens: the 1x1 conv is a GEMM, the permute is free
        for blk in self.transformer_blocks:
            h = blk.run(h, context, kv_bias, checkpoint)
        return g.proj_out([h], residual=alias)


class Downsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)
        self.__dict__["_g"] = None

    def _group(self) -> ConvGroup:
        if self.__dict__["_g"] is None:
            self.__dict__["_g"] = ConvGroup(self.conv)
        g = self.__dict__["_g"]
        g.conv = self.conv
        return g

    def run(self, x, geom):
        return self._group()(x, geom)


class Upsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=1, padding=1)
        self.__dict__["_g"] = None

    def _group(self) -> ConvGroup:
        if self.__dict__["_g"] is None:
            self.__dict__["_g"] = ConvGroup(self.conv)
        g = self.__dict__["_g"]
        g.conv = self.conv
        return g

    def run(self, x, geom):
        B, H, W = geom
        up = ops.Upsample2xFn.apply(geom, x)
        return self._group()(up, (B, 2 * H, 2 * W))


class DownBlock(nn.Module):
    """CrossAttnDownBlock2D / DownBlock2D (has_attn False): resnets [+ attentions] [+ downsamplers]."""

    def __init__(self, cin, cout, temb, n_layers, has_attn, heads, ctx_dim, add_down, groups, depth=1, linear_proj=False):
        super().__init__()
        if has_attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, ctx_dim, groups, depth=depth, use_linear_projection=linear_proj)
                                             for _ in range(n_layers)])
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups) for i in range(n_layers)])
        if add_down:
            self.downsamplers = nn.ModuleList([Downsample2D(cout)])
        self.has_attn, self.gradient_checkpointing = has_attn, False


class MidBlock(nn.Module):
    def __init__(self, ch, temb, heads, ctx_dim, groups, depth=1, linear_proj=False):
        super().__init__()
        self.attentions = nn.ModuleList([Transformer2DModel(ch, heads, ctx_dim, groups, depth=depth, use_linear_projection=linear_proj)])
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb, groups), ResnetBlock2D(ch, ch, temb, groups)])
        self.gradient_checkpointing = False


class UpBlock(nn.Module):
    def __init__(self, in_chs: Sequence[Tuple[int, int]], cout, temb, has_attn, heads, ctx_dim, add_up, groups, depth=1, linear_proj=False):
        super().__init__()
        if has_attn:
            self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, ctx_dim, groups, depth=depth, use_linear_projection=linear_proj)
                                             for _ in in_chs])
        self.resnets = nn.ModuleList([ResnetBlock2D(a + b, cout, temb, groups) for a, b in in_chs])
        for r, split in zip(self.resnets, in_chs):
            r.in_split = tuple(split)
        if add_up:
            self.upsamplers = nn.ModuleList([Upsample2D(cout)])
        self.has_attn, self.gradient_checkpointing = has_attn, False


class UNet2DConditionModel(nn.Module):
    def __init__(self, sample_size: int = 64, in_channels: int = 4, out_channels: int = 4,
                 block_out_channels: Sequence[int] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 attention_head_dim=8, cross_attention_dim: int = 768, norm_num_groups: int = 32,
                 down_block_types: Sequence[str] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                 up_block_types: Sequence[str] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
                 transformer_layers_per_block=1, use_linear_projection: bool = False, addition_embed_type: Optional[str] = None,
                 addition_time_embed_dim: Optional[int] = None, projection_class_embeddings_input_dim: Optional[int] = None,
                 **unused):
        """Constructor keys of the diffusers config.  Defaults = SD1.x (reference cfgs/unet_struct.txt); the SDXL-base config
        (3 levels, `attention_head_dim` (5, 10, 20) = heads per level, `transformer_layers_per_block` (1, 2, 10),
        `use_linear_projection`, `addition_embed_type='text_time'`, 2048-wide context) builds the SDXL UNet the reference reaches
        through hcpdiff/models/wrapper.py:57-75."""
        super().__init__()
        ch = tuple(block_out_channels)
        nlev = len(ch)
        per_level = lambda v: tuple(v) if isinstance(v, (list, tuple)) else (v,) * nlev   # noqa: E731
        heads = per_level(attention_head_dim)       # SD quirk: `attention_head_dim` is the number of heads
        depth = per_level(transformer_layers_per_block)
        if len(down_block_types) != nlev or len(up_block_types) != nlev:
            raise ValueError("down_block_types / up_block_types must have one entry per level")
        if addition_embed_type not in (None, "text_time"):
            raise NotImplementedError(f"addition_embed_type={addition_embed_type!r} is not supported")
        temb = ch[0] * 4
        self.config = SimpleNamespace(sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
                                      block_out_channels=ch, layers_per_block=layers_per_block, attention_head_dim=attention_head_dim,
                                      cross_attention_dim=cross_attention_dim, norm_num_groups=norm_num_groups,
                                      down_block_types=tuple(down_block_types), up_block_types=tuple(up_block_types),
                                      transformer_layers_per_block=transformer_layers_per_block,
                                      use_linear_projection=use_linear_projection, addition_embed_type=addition_embed_type,
                                      addition_time_embed_dim=addition_time_embed_dim,
                                      projection_class_embeddings_input_dim=projection_class_embeddings_input_dim)
        self.conv_in = nn.Conv2d(in_channels, ch[0], 3, padding=1)
        self.time_proj = Timesteps(ch[0])
        self.time_embedding = TimestepEmbedding(ch[0], temb)
        if addition_embed_type == "text_time":
            self.add_time_proj = Timesteps(addition_time_embed_dim)
            self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, temb)
        g = norm_num_groups
        lin = use_linear_projection
        self.down_blocks = nn.ModuleList()
        skip_ch = [ch[0]]
        cprev = ch[0]
        for i, c in enumerate(ch):
            has_attn = down_block_types[i].startswith("CrossAttn")
            last = i == nlev - 1
            self.down_blocks.append(DownBlock(cprev, c, temb, layers_per_block, has_attn, heads[i], cross_attention_dim, not last, g,
                                              depth=depth[i], linear_proj=lin))
            skip_ch += [c] * layers_per_block + ([] if last else [c])
            cprev = c
        self.mid_block = MidBlock(ch[-1], temb, heads[-1], cross_attention_dim, g, depth=depth[-1], linear_proj=lin)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        cprev = ch[-1]
        for i, c in enumerate(rev):
            has_attn = up_block_types[i].startswith("CrossAttn")
            in_chs = []
            for _ in range(layers_per_block + 1):
                in_chs.append((cprev, skip_ch.pop()))
                cprev = c
            self.up_blocks.append(UpBlock(in_chs, c, temb, has_attn, heads[nlev - 1 - i], cross_attention_dim, i < nlev - 1, g,
                                          depth=depth[nlev - 1 - i], linear_proj=lin))
        self.conv_norm_out = nn.GroupNorm(g, ch[0], eps=1e-5)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(ch[0], out_channels, 3, padding=1)
        self.gradient_checkpointing = False
        self.__dict__["_rt"] = None

    # ---- the slice of the diffusers ModelMixin API the reference touches --------------------------------------------
    @property
    def dtype(self) -> torch.dtype:
        return self.conv_in.weight.dtype

    @property
    def device(self) -> torch.device:
        return self.conv_in.weight.device

    def enable_gradient_checkpointing(self):
        """Recompute every BasicTransformerBlock in the backward instead of keeping its intermediates (the reference turns this on
        with `model.gradient_checkpointing`, cfgs/train/train_base.yaml:69).

        With the flag set, a training forward keeps per block only its input, its two attention outputs and their LSE rows; the
        backward reruns the block's LayerNorms and linears on the same kernels (the attention forward is not rerun, the
        feed-forward out-projection's GEMM only when merged LoRA rank rows ride it) and then runs the block's backward.  Results are
        bit-identical to the flag off.  ResnetBlocks, the Transformer2DModel's GroupNorm / proj_in / proj_out, the time embedding and
        the text encoder keep their activations.  The flag costs the recompute's time and lowers the activation memory of each image,
        which lets larger batches fit; it has no effect without grad mode."""
        self.gradient_checkpointing = True

    def enable_xformers_memory_efficient_attention(self, *args, **kwargs):
        """No-op: attention always runs the fused wgmma kernel (reference hcpdiff/train_ac.py:258-263 toggles xFormers here)."""

    def resnets_in_order(self) -> List[ResnetBlock2D]:
        out = []
        for b in self.down_blocks:
            out += list(b.resnets)
        out += list(self.mid_block.resnets)
        for b in self.up_blocks:
            out += list(b.resnets)
        return out

    def linear_groups(self) -> List[LinearGroup]:
        out = []
        for m in self.modules():
            if isinstance(m, (Attention, FeedForward, Transformer2DModel)):
                out += m.linear_groups()
            elif isinstance(m, ResnetBlock2D):
                g = m._groups()
                if g.shortcut is not None:
                    out.append(g.shortcut)
        return out

    def conv_groups(self) -> List[ConvGroup]:
        out = []
        for m in self.modules():
            if isinstance(m, ResnetBlock2D):
                g = m._groups()
                out += [g.conv1, g.conv2]
            elif isinstance(m, (Downsample2D, Upsample2D)):
                out.append(m._group())
        return out

    # ---- time embedding: three skinny-linear launches for the whole network --------------------------------------------
    @staticmethod
    def _temb_host(r) -> nn.Linear:
        """`time_emb_proj` of a resnet, or the host below a LoraPatchContainer patched onto it (`layers: ['re:.*\\.resnets$']`
        wraps every nn.Linear / nn.Conv2d of a ResnetBlock2D, reference cfgs/train/examples/locon.yaml)."""
        m = r.time_emb_proj
        return m._host if hasattr(m, "_host") else m

    def _time_runtime(self):
        rt = self.__dict__["_rt"]
        resnets = self.resnets_in_order()
        te = self.time_embedding
        sig = (te.linear_1.weight._version, te.linear_2.weight._version, te.linear_1.weight.data_ptr(),
               tuple((self._temb_host(r).weight._version, self._temb_host(r).weight.data_ptr(), self._temb_host(r).weight.requires_grad,
                      id(r.time_emb_proj), tuple(getattr(r.time_emb_proj, "plugin_names", ()))) for r in resnets),
               te.linear_1.weight.requires_grad, te.linear_2.weight.requires_grad, self.conv_in.weight.requires_grad,
               self.conv_out.weight.requires_grad, self.conv_in.weight.data_ptr(), self.conv_out.weight.data_ptr(),
               tuple((lin.weight.requires_grad, lin.bias.requires_grad, lin.weight.data_ptr()) for lin in
                     ((self.add_embedding.linear_1, self.add_embedding.linear_2) if hasattr(self, "add_embedding") else ())))
        if rt is None or rt.sig != sig:
            from .lora import DAPPPatchContainer, LoraPatchContainer
            for p in (te.linear_1, te.linear_2):
                if not isinstance(p, nn.Linear):
                    raise NotImplementedError("plugins on time_embedding.linear_1 / linear_2 are not supported on the H100 hot path")
            for r in resnets:
                m = r.time_emb_proj
                if isinstance(m, DAPPPatchContainer) or not isinstance(m, (nn.Linear, LoraPatchContainer)):
                    raise NotImplementedError(f"{type(m).__name__} on time_emb_proj is not supported on the H100 hot path")
            rt = SimpleNamespace(sig=sig)
            # LoRA on time_emb_proj: per patched resnet the stacked blocks; their rank-r products are two small fp32 linears each
            rt.temb_lora = [[m[name] for name in m.plugin_names] if isinstance(m, LoraPatchContainer) else []
                            for m in (r.time_emb_proj for r in resnets)]
            for blocks in rt.temb_lora:
                for b in blocks:
                    if b.rank % 2 or (b.dropout.p > 0 and b.dropout.training):
                        raise NotImplementedError("LoRA on time_emb_proj needs an even rank and dropout 0")
            # full fine-tune: the time-embedding MLP, the time_emb_proj layers and the boundary convolutions are trained -> their
            # operands are refreshed every step and the path records autograd nodes (ops.SmallLinearFn / ConvInFn / ConvOutFn)
            rt.train_time = any(p.weight.requires_grad for p in (te.linear_1, te.linear_2, *[self._temb_host(r) for r in resnets]))
            rt.train_in, rt.train_out = self.conv_in.weight.requires_grad, self.conv_out.weight.requires_grad
            rt.w1 = te.linear_1.weight.detach().to(torch.bfloat16).contiguous()
            rt.b1 = te.linear_1.bias.detach().float().contiguous()
            rt.w2 = te.linear_2.weight.detach().to(torch.bfloat16).contiguous()
            rt.b2 = te.linear_2.bias.detach().float().contiguous()
            rt.add = None
            rt.add_unfused = False
            if hasattr(self, "add_embedding"):
                ae = self.add_embedding
                for p in (ae.linear_1, ae.linear_2):
                    if not isinstance(p, nn.Linear):
                        raise NotImplementedError("plugins on the additional-embedding layers are not supported on the H100 hot path")
                train_add = any(q.requires_grad for lin in (ae.linear_1, ae.linear_2) for q in (lin.weight, lin.bias))
                rt.add_unfused = rt.train_time or train_add
            if rt.add_unfused:
                # training (full fine-tune of an SDXL UNet): emb = silu(linear_2(e1) + add_embedding.linear_2(a1)) as two small
                # linears with autograd nodes; the trained add-embedding operands are refreshed every step like the time MLP's
                rt.add = SimpleNamespace(
                    w1=ae.linear_1.weight.detach().to(torch.bfloat16).contiguous(), b1=ae.linear_1.bias.detach().float().clone(),
                    w2=ae.linear_2.weight.detach().to(torch.bfloat16).contiguous(), b2=ae.linear_2.bias.detach().float().clone(),
                    l1=[(ae.linear_1.weight, ae.linear_1.bias, 0, ae.linear_1.weight.shape[0])] if train_add else None,
                    l2=[(ae.linear_2.weight, ae.linear_2.bias, 0, ae.linear_2.weight.shape[0])] if train_add else None)
            elif hasattr(self, "add_embedding"):
                # emb = time_embedding(t) + add_embedding(cat[text_embeds, sinusoid(time_ids)]): the two second linears are one
                # skinny GEMM over the concatenated hidden vectors [e1 | a1] with W = [W2 | Wa2], b = b2 + ba2
                rt.add = SimpleNamespace(
                    w1=ae.linear_1.weight.detach().to(torch.bfloat16).contiguous(), b1=ae.linear_1.bias.detach().float().contiguous(),
                    w2cat=torch.cat([te.linear_2.weight.detach(), ae.linear_2.weight.detach()], 1).to(torch.bfloat16).contiguous(),
                    b2sum=(te.linear_2.bias.detach() + ae.linear_2.bias.detach()).float().contiguous(),
                    # the unfused operands, for a text_embeds that carries a gradient (a trained text encoder in front)
                    w2=ae.linear_2.weight.detach().to(torch.bfloat16).contiguous(), b2=ae.linear_2.bias.detach().float().contiguous(),
                    l1=None, l2=None)
            rt.wp = torch.cat([self._temb_host(r).weight.detach() for r in resnets], 0).to(torch.bfloat16).contiguous()
            rt.bp = torch.cat([self._temb_host(r).bias.detach() for r in resnets], 0).float().contiguous()
            offs, o = [], 0
            for r in resnets:
                offs.append((o, o + r.out_channels))
                o += r.out_channels
            rt.offs = offs
            rt.repack = _JobTable()
            rt.time_jobs = []

            def job(kind, src, dst, rows, K, o0):
                j = _lib.RepackJob()
                j.src, j.dst0, j.dst1 = src.data_ptr(), dst.data_ptr(), None
                j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = kind, rows, K, o0, 0, 0
                return j
            if rt.train_time:
                for lin, wdst, bdst in ((te.linear_1, rt.w1, rt.b1), (te.linear_2, rt.w2, rt.b2)):
                    rt.time_jobs += [job(3, lin.weight, wdst, lin.weight.shape[0], lin.weight.shape[1], 0),
                                     job(2, lin.bias, bdst, lin.bias.shape[0], 1, 0)]
                for r, (a, b) in zip(resnets, offs):
                    tp = self._temb_host(r)
                    rt.time_jobs += [job(3, tp.weight, rt.wp, b - a, tp.weight.shape[1], a), job(2, tp.bias, rt.bp, b - a, 1, a)]
                # b1 / b2 must be own buffers (a .float() of an fp32 parameter is the parameter itself)
                rt.b1, rt.b2 = rt.b1.clone(), rt.b2.clone()
                rt.time_jobs[1].dst0, rt.time_jobs[3].dst0 = rt.b1.data_ptr(), rt.b2.data_ptr()
                rt.train_lists = SimpleNamespace(
                    l1=[(te.linear_1.weight, te.linear_1.bias, 0, te.linear_1.weight.shape[0])],
                    l2=[(te.linear_2.weight, te.linear_2.bias, 0, te.linear_2.weight.shape[0])],
                    proj=[(self._temb_host(r).weight, self._temb_host(r).bias, a, b - a) for r, (a, b) in zip(resnets, offs)])
            if rt.add_unfused and rt.add.l1 is not None:
                for lin, wdst, bdst in ((ae.linear_1, rt.add.w1, rt.add.b1), (ae.linear_2, rt.add.w2, rt.add.b2)):
                    rt.time_jobs += [job(3, lin.weight, wdst, lin.weight.shape[0], lin.weight.shape[1], 0),
                                     job(2, lin.bias, bdst, lin.bias.shape[0], 1, 0)]
            rt.w_in = self.conv_in.weight.detach().float().permute(1, 2, 3, 0).contiguous()       # tap-major [Cin,3,3,Cout]
            rt.b_in = self.conv_in.bias.detach().float().contiguous()
            rt.w_out = self.conv_out.weight.detach().float().permute(2, 3, 0, 1).contiguous()     # tap-major [3,3,Cout,Cin]
            rt.b_out = self.conv_out.bias.detach().float().contiguous()
            rt.jobs = _JobTable()
            self.__dict__["_rt"] = rt
        return rt

    def _add_input(self, added, B, dev) -> torch.Tensor:
        """cat[text_embeds, sinusoid(time_ids)] [B, projection_class_embeddings_input_dim], fp32 (the add_embedding input)."""
        te_, ids = added["text_embeds"], added["time_ids"]
        cfg = self.config
        P_, D_ = cfg.projection_class_embeddings_input_dim, cfg.addition_time_embed_dim
        n_ids = ids.shape[-1]
        if te_.shape[-1] + n_ids * D_ != P_:
            raise ValueError(f"text_embeds ({te_.shape[-1]}) + time_ids ({n_ids} x {D_}) do not add up to {P_}")
        addin = torch.empty((B, P_), dtype=torch.float32, device=dev)
        addin[:, :te_.shape[-1]].copy_(te_)                           # boundary copy; the sinusoids are written next to it
        ops.sinusoid(ids.to(dev, torch.float32).reshape(-1).contiguous(), D_, n_ids, addin, te_.shape[-1])
        return addin

    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor,
                encoder_attention_mask: Optional[torch.Tensor] = None, return_dict: bool = True, **kwargs):
        if not sample.is_cuda:
            raise _lib.HcpError("hcp_diffusion_b200.UNet2DConditionModel runs on a CUDA (sm_90) device only; there is no CPU fallback")
        for key in ("class_labels", "down_block_additional_residuals", "mid_block_additional_residual"):
            if kwargs.get(key) is not None:
                raise NotImplementedError(f"`{key}` is not supported by the hot path")
        added = kwargs.get("added_cond_kwargs")
        if hasattr(self, "add_embedding"):
            if not added or "text_embeds" not in added or "time_ids" not in added:
                raise ValueError("this UNet has addition_embed_type='text_time': pass added_cond_kwargs={'text_embeds', 'time_ids'} "
                                 "(reference hcpdiff/models/wrapper.py:66)")
        elif added:
            raise NotImplementedError("`added_cond_kwargs` given to a UNet without an additional embedding")
        B, _, H, W = sample.shape
        nlev = len(self.config.block_out_channels)
        if H % (1 << (nlev - 1)) or W % (1 << (nlev - 1)):
            raise ValueError("latent height/width must be divisible by 2^(num_blocks-1)")
        rt = self._time_runtime()
        dev = sample.device

        # LoRA operands: every group is (re)built if stale, then ONE launch re-packs all low-rank factors from the fp32 params
        groups = self.linear_groups()
        for g in groups:
            g.prepare(g._k_splits)
        cgroups = self.conv_groups()
        for g in cgroups:
            g.prepare()
        pack_lora(groups + cgroups, rt.jobs)
        # full fine-tune: one launch re-casts every trained fp32 master into the kernels' bf16 operand layouts
        repack_trained(groups + cgroups, rt.repack, rt.time_jobs)
        if rt.train_in:
            rt.w_in = self.conv_in.weight.detach().float().permute(1, 2, 3, 0).contiguous()
            rt.b_in = self.conv_in.bias.detach().float().contiguous()
        if rt.train_out:
            rt.w_out = self.conv_out.weight.detach().float().permute(2, 3, 0, 1).contiguous()
            rt.b_out = self.conv_out.bias.detach().float().contiguous()

        # time embedding -> per-resnet bias rows [B, sum(C)] fp32
        t = torch.as_tensor(timestep, device=dev)
        if t.dim() == 0:
            t = t[None]
        t = t.expand(B).to(torch.float32).contiguous()
        # d(text_embeds) wanted (SDXL with a trained text encoder, whose pooled projection is text_embeds): the unfused path, whose
        # add_embedding.linear_1 node produces dx; a frozen add_embedding stays frozen
        te_grad = rt.add is not None and added["text_embeds"].requires_grad and torch.is_grad_enabled()
        unfused = rt.add_unfused or te_grad
        if unfused:
            x0 = torch.empty((B, self.time_proj.num_channels), dtype=torch.float32, device=dev)
            ops.sinusoid(t, self.time_proj.num_channels, 1, x0, 0)
            lists = rt.train_lists if rt.train_time else None
            e1 = ops.small_linear(x0, rt.w1, rt.b1, True, lists and lists.l1)
            a1 = ops.small_linear(self._add_input(added, B, dev), rt.add.w1, rt.add.b1, True, rt.add.l1)
            z = ops.small_linear(e1, rt.w2, rt.b2, False, lists and lists.l2) + ops.small_linear(a1, rt.add.w2, rt.add.b2, False, rt.add.l2)
            emb = ops.silu(z)
        elif rt.train_time:
            x0 = torch.empty((B, self.time_proj.num_channels), dtype=torch.float32, device=dev)
            ops.sinusoid(t, self.time_proj.num_channels, 1, x0, 0)
            e1 = ops.small_linear(x0, rt.w1, rt.b1, True, rt.train_lists.l1)
            emb = ops.small_linear(e1, rt.w2, rt.b2, True, rt.train_lists.l2)
        elif rt.add is None:
            e1 = ops.skinny_linear(t, rt.w1, rt.b1, 2, True)             # silu(linear_1(sinusoid(t)))
            emb = ops.skinny_linear(e1, rt.w2, rt.b2, 0, True)           # silu(linear_2(.)): every consumer applies SiLU first
        else:
            e1 = ops.skinny_linear(t, rt.w1, rt.b1, 2, True)
            a1 = ops.skinny_linear(self._add_input(added, B, dev), rt.add.w1, rt.add.b1, 0, True)  # silu(add_embedding.linear_1(.))
            emb = ops.skinny_linear(torch.cat([e1, a1], 1), rt.add.w2cat, rt.add.b2sum, 0, True)   # silu(linear_2(e1) + add.linear_2(a1))
        if rt.train_time or unfused:
            # an autograd node whenever emb carries a gradient: the trained add_embedding needs dL/demb even when every
            # time_emb_proj is frozen
            temb_all = ops.small_linear(emb, rt.wp, rt.bp, False, rt.train_lists.proj if rt.train_time else None)
        else:
            temb_all = ops.skinny_linear(emb, rt.wp, rt.bp, 0, False)    # all 22 time_emb_proj layers at once
        temb_list = [temb_all[:, a:b] for a, b in rt.offs]
        for i, blocks in enumerate(rt.temb_lora):
            # y = x (W + sum alpha B A)^T + b on the M = batch rows of the time embedding: T = emb A^T, delta = alpha T B^T
            for b in blocks:
                T = ops.small_linear(emb, b.layer.W_down.detach().to(torch.bfloat16), None, False, [(b.layer.W_down, None, 0, b.rank)])
                d = ops.small_linear(T, b.layer.W_up.detach().to(torch.bfloat16), None, False, [(b.layer.W_up, None, 0, b.layer.W_up.shape[0])])
                temb_list[i] = temb_list[i] + d * b.alpha
        tembs = iter(temb_list)

        attn2s = [m.attn2 for m in self.modules() if isinstance(m, BasicTransformerBlock)]
        if encoder_hidden_states.requires_grad and torch.is_grad_enabled():
            # d(ehs): every cross-attention's k/v dgrad (merged LoRA included) summed in fp32; without a gradient nothing changes
            ctx = _PerAttnContext(encoder_hidden_states, attn2s)
        else:
            ctx = ops.cast_bf16(encoder_hidden_states)
        ckpt = self.gradient_checkpointing and torch.is_grad_enabled()
        kv_bias = None
        if encoder_attention_mask is not None:
            kv_bias = ((1.0 - encoder_attention_mask.to(torch.float32)) * -10000.0).contiguous()

        if ops.side_enabled():
            ctx = _HoistedKV(ctx, attn2s)

        h = ops.conv_in(sample, rt.w_in, rt.b_in,                        # bf16 [B, H*W, C0]
                        train=(self.conv_in.weight, self.conv_in.bias) if rt.train_in else None)
        geom = (B, H, W)
        skips: List[Tuple[torch.Tensor, tuple]] = []

        def push(x):
            a, b = ops.Fork2Fn.apply(x) if x.requires_grad else (x, x)
            skips.append(a)
            return b

        h = push(h)
        for blk in self.down_blocks:
            for j, res in enumerate(blk.resnets):
                h = res.run([h], geom, next(tembs))
                if blk.has_attn:
                    h = blk.attentions[j].run(h, ctx, kv_bias, ckpt)
                h = push(h)
            if hasattr(blk, "downsamplers"):
                h = blk.downsamplers[0].run(h, geom)
                geom = (B, geom[1] // 2, geom[2] // 2)
                h = push(h)
        h = self.mid_block.resnets[0].run([h], geom, next(tembs))
        h = self.mid_block.attentions[0].run(h, ctx, kv_bias, ckpt)
        h = self.mid_block.resnets[1].run([h], geom, next(tembs))
        for blk in self.up_blocks:
            for j, res in enumerate(blk.resnets):
                h = res.run([h, skips.pop()], geom, next(tembs))
                if blk.has_attn:
                    h = blk.attentions[j].run(h, ctx, kv_bias, ckpt)
            if hasattr(blk, "upsamplers"):
                h = blk.upsamplers[0].run(h, geom)
                geom = (B, geom[1] * 2, geom[2] * 2)
        n = self.conv_norm_out
        y = ops.group_norm(n.weight, n.bias, n.num_groups, n.eps, True, h, None)[0]
        out = ops.ConvOutFn.apply(rt.w_out, rt.b_out, geom, (self.conv_out.weight, self.conv_out.bias) if rt.train_out else None, y)
        if out.dtype != sample.dtype and sample.dtype.is_floating_point:
            out = out.to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)
