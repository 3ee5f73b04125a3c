"""`CLIPTextModel` (the SD1.x text encoder) executed by the libhcpb200 kernels, and the reference's prompt composition.

Drop-in for the text-encoder seam of the reference trainer: the module tree reproduces transformers' names and parameter shapes
(reference cfgs/te_struct.txt), so a transformers state dict loads strictly and the `lora_text_encoder` regexes of the reference
configs (`re:.*self_attn$`, `re:.*mlp$`) select the same layers.  Every leaf is a real nn.Embedding / nn.Linear / nn.LayerNorm that
hcpdiff's plugin surgery can wrap.  As in the UNet, execution does not go through the leaves' forward(): each encoder layer drives
fused kernels over bf16 token matrices (ops.py) and the fp32 master parameters stay in the modules.

Per layer (pre-LN): LayerNorm -> fused q|k|v GEMM with biases -> causal attention (scale d^-1/2) -> out_proj with the residual in
its epilogue -> LayerNorm -> fc1 -> quick-GELU -> fc2 with the residual in its epilogue.  LoRA adapters ride the linear groups'
merged operands exactly as in the UNet.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Tuple

import torch
from torch import nn

from .. import _lib, ops
from ..runtime import LinearGroup, _JobTable, pack_lora
from .lora import DAPPPatchContainer
from .plugin import BasePluginBlock


@dataclass
class CLIPTextModelOutput:
    """The fields of transformers' BaseModelOutputWithPooling the reference reads (TEEXHook.forward_hook)."""
    last_hidden_state: torch.Tensor
    pooler_output: Optional[torch.Tensor] = None
    hidden_states: Optional[Tuple[torch.Tensor, ...]] = None

    def __getitem__(self, key):
        if isinstance(key, str):
            return getattr(self, key)
        return tuple(v for v in (self.last_hidden_state, self.pooler_output, self.hidden_states) if v is not None)[key]


class QuickGELUActivation(nn.Module):
    """x * sigmoid(1.702 x) (transformers.activations.QuickGELUActivation); runs as hcp_quick_gelu_*_bf16."""


class CLIPTextEmbeddings(nn.Module):
    def __init__(self, vocab_size: int, hidden_size: int, max_position_embeddings: int):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab_size, hidden_size)
        self.position_embedding = nn.Embedding(max_position_embeddings, hidden_size)


class CLIPAttention(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int):
        super().__init__()
        if hidden_size % num_heads:
            raise ValueError(f"hidden_size {hidden_size} is not a multiple of num_attention_heads {num_heads}")
        self.embed_dim, self.num_heads = hidden_size, num_heads
        self.head_dim = hidden_size // num_heads
        self.scale = self.head_dim ** -0.5
        self.k_proj = nn.Linear(hidden_size, hidden_size)
        self.v_proj = nn.Linear(hidden_size, hidden_size)
        self.q_proj = nn.Linear(hidden_size, hidden_size)
        self.out_proj = nn.Linear(hidden_size, hidden_size)
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(qkv=LinearGroup([]), out=LinearGroup([]))
            self.__dict__["_g"] = g
        g.qkv.children = [self.q_proj, self.k_proj, self.v_proj]
        g.out.children = [self.out_proj]
        return g

    def run(self, x: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        g = self._groups()
        C_ = self.embed_dim
        qkv = g.qkv([x])                                                  # [B, L, 3C]: one GEMM with the three biases
        o = ops.attention(self.num_heads, C_, (0, C_, 2 * C_), qkv, None, None, causal=True)
        return g.out([o], residual=residual)


class CLIPMLP(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int):
        super().__init__()
        self.activation_fn = QuickGELUActivation()
        self.fc1 = nn.Linear(hidden_size, intermediate_size)
        self.fc2 = nn.Linear(intermediate_size, hidden_size)
        self.__dict__["_g"] = None

    def _groups(self):
        g = self.__dict__["_g"]
        if g is None:
            g = SimpleNamespace(fc1=LinearGroup([]), fc2=LinearGroup([]))
            self.__dict__["_g"] = g
        g.fc1.children = [self.fc1]
        g.fc2.children = [self.fc2]
        return g

    def run(self, x: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        g = self._groups()
        h = ops.QuickGeluFn.apply(g.fc1([x]))
        return g.fc2([h], residual=residual)


class CLIPEncoderLayer(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, intermediate_size: int, eps: float):
        super().__init__()
        self.self_attn = CLIPAttention(hidden_size, num_heads)
        self.layer_norm1 = nn.LayerNorm(hidden_size, eps=eps)
        self.mlp = CLIPMLP(hidden_size, intermediate_size)
        self.layer_norm2 = nn.LayerNorm(hidden_size, eps=eps)

    def linear_groups(self) -> List[LinearGroup]:
        a, m = self.self_attn._groups(), self.mlp._groups()
        return [a.qkv, a.out, m.fc1, m.fc2]

    def run(self, h: torch.Tensor) -> torch.Tensor:
        n, a = ops.layer_norm(self.layer_norm1.weight, self.layer_norm1.bias, self.layer_norm1.eps, h)
        h = self.self_attn.run(n, a)
        n, a = ops.layer_norm(self.layer_norm2.weight, self.layer_norm2.bias, self.layer_norm2.eps, h)
        return self.mlp.run(n, a)


class CLIPEncoder(nn.Module):
    def __init__(self, n_layers: int, hidden_size: int, num_heads: int, intermediate_size: int, eps: float):
        super().__init__()
        self.layers = nn.ModuleList([CLIPEncoderLayer(hidden_size, num_heads, intermediate_size, eps) for _ in range(n_layers)])


class CLIPTextTransformer(nn.Module):
    def __init__(self, cfg: SimpleNamespace):
        super().__init__()
        self.embeddings = CLIPTextEmbeddings(cfg.vocab_size, cfg.hidden_size, cfg.max_position_embeddings)
        self.encoder = CLIPEncoder(cfg.num_hidden_layers, cfg.hidden_size, cfg.num_attention_heads, cfg.intermediate_size,
                                   cfg.layer_norm_eps)
        self.final_layer_norm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


class CLIPTextModel(nn.Module):
    def __init__(self, vocab_size: int = 49408, hidden_size: int = 768, intermediate_size: int = 3072, num_hidden_layers: int = 12,
                 num_attention_heads: int = 12, max_position_embeddings: int = 77, hidden_act: str = "quick_gelu",
                 layer_norm_eps: float = 1e-5, pad_token_id: int = 1, bos_token_id: int = 49406, eos_token_id: int = 49407, **unused):
        """Constructor keys of `transformers.CLIPTextConfig`; the defaults build the SD1.x text encoder (CLIP ViT-L/14, reference
        cfgs/te_struct.txt, 123,060,480 parameters)."""
        super().__init__()
        if hidden_act != "quick_gelu":
            raise NotImplementedError(f"hidden_act={hidden_act!r}: only quick_gelu (the SD1.x text encoder) is supported")
        self.config = SimpleNamespace(vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
                                      num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                                      max_position_embeddings=max_position_embeddings, hidden_act=hidden_act,
                                      layer_norm_eps=layer_norm_eps, pad_token_id=pad_token_id, bos_token_id=bos_token_id,
                                      eos_token_id=eos_token_id)
        self.text_model = CLIPTextTransformer(self.config)
        self.__dict__["_jobs"] = _JobTable()

    @property
    def dtype(self) -> torch.dtype:
        return self.text_model.final_layer_norm.weight.dtype

    @property
    def device(self) -> torch.device:
        return self.text_model.final_layer_norm.weight.device

    def linear_groups(self) -> List[LinearGroup]:
        out = []
        for layer in self.text_model.encoder.layers:
            out += layer.linear_groups()
        return out

    def _check_trainable(self) -> None:
        """Only LoRA adapters train here: a base parameter that requires a gradient (full fine-tune) or a DreamArtist++ container is
        refused instead of being silently frozen."""
        for name, m in self.named_modules():
            if isinstance(m, DAPPPatchContainer):
                raise NotImplementedError(f"DreamArtist++ adapters on the text encoder ({name}) are not supported")
        if not torch.is_grad_enabled():
            return
        plugin_params = {id(p) for m in self.modules() if isinstance(m, BasePluginBlock) for p in m.parameters()}
        for name, p in self.named_parameters():
            if p.requires_grad and id(p) not in plugin_params:
                raise NotImplementedError(f"{name} requires a gradient: full fine-tuning of the text encoder is not supported "
                                          "(freeze the base model with requires_grad_(False); LoRA adapters train)")

    def run_layers(self, input_ids: torch.Tensor, n_layers: int, position_ids: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        """[embeddings, output of layer 1, ..., output of layer n_layers] as bf16 [B, L, C]; only the first n_layers layers run."""
        if not input_ids.is_cuda:
            raise _lib.HcpError("hcp_diffusion_b200.CLIPTextModel runs on a CUDA (sm_90) device only; there is no CPU fallback")
        if input_ids.dim() != 2:
            raise ValueError(f"input_ids must be [batch, tokens], got {tuple(input_ids.shape)}")
        self._check_trainable()
        layers = self.text_model.encoder.layers[:n_layers]
        groups = [g for layer in layers for g in layer.linear_groups()]
        for g in groups:
            g.prepare()
        pack_lora(groups, self.__dict__["_jobs"])
        emb = self.text_model.embeddings
        h = ops.embed_tokens(input_ids.long(), emb.token_embedding.weight, emb.position_embedding.weight, position_ids)
        out = [h]
        for layer in layers:
            h = layer.run(h)
            out.append(h)
        return out

    def final_norm(self, h: torch.Tensor) -> torch.Tensor:
        n = self.text_model.final_layer_norm
        return ops.layer_norm(n.weight, n.bias, n.eps, h)[0]

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                output_hidden_states: bool = False, return_dict: bool = True, **kwargs):
        """transformers' CLIPTextModel.forward: `last_hidden_state` (final LayerNorm), `pooler_output` (the row of the largest id,
        the EOS token of the SD1.x tokenizer), and with output_hidden_states the embeddings plus every layer's output."""
        if attention_mask is not None:
            raise NotImplementedError("attention_mask on the text encoder is not supported (the reference's default "
                                      "use_attention_mask=False never passes one)")
        hs = self.run_layers(input_ids, len(self.text_model.encoder.layers), position_ids)
        last = self.final_norm(hs[-1])
        pooled = last[torch.arange(last.shape[0], device=last.device), input_ids.to(last.device).argmax(-1)]
        out = CLIPTextModelOutput(last_hidden_state=last, pooler_output=pooled, hidden_states=tuple(hs) if output_hidden_states else None)
        return out if return_dict else out[:]


def encode_prompt(te: CLIPTextModel, input_ids: torch.Tensor, n_repeats: int = 1, clip_skip: int = 0,
                  clip_final_norm: bool = True) -> torch.Tensor:
    """The reference's TEEXHook composition (hcpdiff/models/textencoder_ex.py:60-82) around the text encoder: ids [B, 77 R] are
    encoded as B R prompts of 77 tokens, the hidden state `clip_skip` layers before the last is taken (final LayerNorm applied when
    `clip_final_norm`), and the R chunks are rejoined as BOS + R x 75 middle rows + EOS -> bf16 [B, 75 R + 2, C].

    Only the first num_hidden_layers - clip_skip layers run.  The reference keeps the skipped layers in its graph with gradient 0; here
    their adapters receive no gradient contribution.  In `LoraTrainStep` their gradients live in the flat buffer, which is zeroed
    every step, so they get the reference's zero gradient and AdamW still decays them."""
    n_total = len(te.text_model.encoder.layers)
    if not 0 <= clip_skip < n_total:
        raise ValueError(f"clip_skip must be in [0, {n_total})")
    B, LR = input_ids.shape
    if LR % n_repeats:
        raise ValueError(f"input_ids width {LR} is not a multiple of n_repeats={n_repeats}")
    L = LR // n_repeats
    ids = input_ids.reshape(B * n_repeats, L)
    h = te.run_layers(ids, n_total - clip_skip)[-1]
    if clip_final_norm:
        h = te.final_norm(h)
    h = h.view(B, n_repeats, L, h.shape[-1])
    # row gathers only (copies): BOS of the first chunk, the middle rows of every chunk, EOS of the last chunk
    return torch.cat([h[:, 0, :1], h[:, :, 1:-1].flatten(1, 2), h[:, -1, -1:]], dim=1)
