"""`CLIPTextModel` (the SD1.x text encoder), `CLIPTextModelWithProjection` and `SDXLTextEncoder` (SDXL's pair) executed by the
libhcpb200 kernels, and the reference's prompt composition.

Drop-in for the text-encoder seam of the reference trainer: the module tree reproduces transformers' names and parameter shapes
(reference cfgs/te_struct.txt), so a transformers state dict loads strictly and the `lora_text_encoder` regexes of the reference
configs (`re:.*self_attn$`, `re:.*mlp$`) select the same layers.  Every leaf is a real nn.Embedding / nn.Linear / nn.LayerNorm that
hcpdiff's plugin surgery can wrap.  As in the UNet, execution does not go through the leaves' forward(): each encoder layer drives
fused kernels over bf16 token matrices (ops.py) and the fp32 master parameters stay in the modules.

Per layer (pre-LN): LayerNorm -> fused q|k|v GEMM with biases -> causal attention (scale d^-1/2) -> out_proj with the residual in
its epilogue -> LayerNorm -> fc1 -> quick-GELU (exact GELU in OpenCLIP-bigG) -> fc2 with the residual in its epilogue.  LoRA adapters
ride the linear groups' merged operands exactly as in the UNet.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Tuple

import torch
from torch import nn

from .. import _lib, ops
from ..runtime import LinearGroup, _JobTable, pack_lora, repack_trained
from .lora import DAPPPatchContainer


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


class GELUActivation(nn.Module):
    """0.5 x (1 + erf(x / sqrt 2)) (transformers.activations.GELUActivation, hidden_act='gelu'); runs as hcp_gelu_*_bf16."""


_ACTIVATIONS = {"quick_gelu": (QuickGELUActivation, ops.QuickGeluFn), "gelu": (GELUActivation, ops.GeluFn)}


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
    def __init__(self, hidden_size: int, intermediate_size: int, hidden_act: str = "quick_gelu"):
        super().__init__()
        module, self.__dict__["_act"] = _ACTIVATIONS[hidden_act]
        self.activation_fn = module()
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
        h = self.__dict__["_act"].apply(g.fc1([x]))
        return g.fc2([h], residual=residual)


class CLIPEncoderLayer(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, intermediate_size: int, eps: float, hidden_act: str = "quick_gelu"):
        super().__init__()
        self.self_attn = CLIPAttention(hidden_size, num_heads)
        self.layer_norm1 = nn.LayerNorm(hidden_size, eps=eps)
        self.mlp = CLIPMLP(hidden_size, intermediate_size, hidden_act)
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
    def __init__(self, n_layers: int, hidden_size: int, num_heads: int, intermediate_size: int, eps: float, hidden_act: str = "quick_gelu"):
        super().__init__()
        self.layers = nn.ModuleList([CLIPEncoderLayer(hidden_size, num_heads, intermediate_size, eps, hidden_act) for _ in range(n_layers)])


class CLIPTextTransformer(nn.Module):
    def __init__(self, cfg: SimpleNamespace):
        super().__init__()
        self.embeddings = CLIPTextEmbeddings(cfg.vocab_size, cfg.hidden_size, cfg.max_position_embeddings)
        self.encoder = CLIPEncoder(cfg.num_hidden_layers, cfg.hidden_size, cfg.num_attention_heads, cfg.intermediate_size,
                                   cfg.layer_norm_eps, cfg.hidden_act)
        self.final_layer_norm = nn.LayerNorm(cfg.hidden_size, eps=cfg.layer_norm_eps)


class CLIPTextModel(nn.Module):
    _hidden_acts = ("quick_gelu",)

    def __init__(self, vocab_size: int = 49408, hidden_size: int = 768, intermediate_size: int = 3072, num_hidden_layers: int = 12,
                 num_attention_heads: int = 12, max_position_embeddings: int = 77, hidden_act: str = "quick_gelu",
                 layer_norm_eps: float = 1e-5, pad_token_id: int = 1, bos_token_id: int = 49406, eos_token_id: int = 49407, **unused):
        """Constructor keys of `transformers.CLIPTextConfig`; the defaults build the SD1.x text encoder (CLIP ViT-L/14, reference
        cfgs/te_struct.txt, 123,060,480 parameters)."""
        super().__init__()
        if hidden_act not in self._hidden_acts:
            raise NotImplementedError(f"hidden_act={hidden_act!r}: {type(self).__name__} supports {' / '.join(self._hidden_acts)} "
                                      "(the exact-GELU encoder is SDXL's second one, CLIPTextModelWithProjection)")
        self.config = SimpleNamespace(vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
                                      num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                                      max_position_embeddings=max_position_embeddings, hidden_act=hidden_act,
                                      layer_norm_eps=layer_norm_eps, pad_token_id=pad_token_id, bos_token_id=bos_token_id,
                                      eos_token_id=eos_token_id)
        self.text_model = CLIPTextTransformer(self.config)
        self.__dict__["_jobs"] = _JobTable()
        self.__dict__["_repack"] = _JobTable()

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
        """LoRA adapters and base parameters (the `text_encoder:` full fine-tune list) train; a DreamArtist++ container is refused
        instead of being silently run as a plain LoRA."""
        for name, m in self.named_modules():
            if isinstance(m, DAPPPatchContainer):
                raise NotImplementedError(f"DreamArtist++ adapters on the text encoder ({name}) are not supported")

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
        # full fine-tune: one launch re-casts the trained fp32 masters the optimizer updated into the GEMMs' bf16 operands
        repack_trained(groups, self.__dict__["_repack"])
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
    their adapters (and, under full fine-tuning, their base parameters) receive no gradient contribution.  In `LoraTrainStep` their
    gradients live in the flat buffer, which is zeroed every step, so they get the reference's zero gradient and AdamW still decays
    them."""
    n_total = len(te.text_model.encoder.layers)
    if not 0 <= clip_skip < n_total:
        raise ValueError(f"clip_skip must be in [0, {n_total})")
    B, LR = input_ids.shape
    if LR % n_repeats:
        raise ValueError(f"input_ids width {LR} is not a multiple of n_repeats={n_repeats}")
    L = LR // n_repeats
    ids = input_ids.reshape(B * n_repeats, L)
    return _compose(te, te.run_layers(ids, n_total - clip_skip)[-1], B, n_repeats, clip_final_norm)


def _compose(te: CLIPTextModel, h: torch.Tensor, B: int, n_repeats: int, clip_final_norm: bool) -> torch.Tensor:
    """The taken hidden state [B R, L, C] -> [B, 75 R + 2, C] (TEEXHook.forward_hook after the hidden-state pick)."""
    if clip_final_norm:
        h = te.final_norm(h)
    h = h.view(B, n_repeats, h.shape[1], h.shape[-1])
    # row gathers only (copies): BOS of the first chunk, the middle rows of every chunk, EOS of the last chunk
    return torch.cat([h[:, 0, :1], h[:, :, 1:-1].flatten(1, 2), h[:, -1, -1:]], dim=1)


class CLIPTextModelWithProjection(CLIPTextModel):
    """transformers.CLIPTextModelWithProjection: the text model plus the bias-free `text_projection` of the pooled row.  The defaults
    build SDXL's second text encoder (OpenCLIP ViT-bigG/14: 1280 wide, 32 layers of 20 heads, exact-GELU MLP, projection 1280), so
    the state dict of stable-diffusion-xl-base-1.0's `text_encoder_2` loads strictly.  `pooler_output` is `text_embeds`, as in the
    reference's CLIPTextModelWithProjection_Align (hcpdiff/models/compose/sdxl_composer.py).

    `text_projection` runs as a LinearGroup (a GEMM at every batch size, plugins wrap it like any other nn.Linear)."""
    _hidden_acts = ("gelu", "quick_gelu")

    def __init__(self, vocab_size: int = 49408, hidden_size: int = 1280, intermediate_size: int = 5120, num_hidden_layers: int = 32,
                 num_attention_heads: int = 20, max_position_embeddings: int = 77, hidden_act: str = "gelu", layer_norm_eps: float = 1e-5,
                 projection_dim: int = 1280, pad_token_id: int = 1, bos_token_id: int = 0, eos_token_id: int = 2, **unused):
        super().__init__(vocab_size=vocab_size, hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         max_position_embeddings=max_position_embeddings, hidden_act=hidden_act, layer_norm_eps=layer_norm_eps,
                         pad_token_id=pad_token_id, bos_token_id=bos_token_id, eos_token_id=eos_token_id)
        self.config.projection_dim = projection_dim
        self.text_projection = nn.Linear(hidden_size, projection_dim, bias=False)
        self.__dict__["_proj"] = LinearGroup([])
        self.__dict__["_proj_jobs"] = _JobTable()
        self.__dict__["_proj_repack"] = _JobTable()

    def linear_groups(self) -> List[LinearGroup]:
        return super().linear_groups() + [self._proj_group()]

    def _proj_group(self) -> LinearGroup:
        g = self.__dict__["_proj"]
        g.children = [self.text_projection]
        return g

    def project(self, last: torch.Tensor, input_ids: torch.Tensor) -> torch.Tensor:
        """text_projection(last[b, argmax(ids[b])]) -> fp32 [B, projection_dim]; `last` is the final-normed last hidden state.  The row
        of the largest id is the first EOS 49407 whether the prompt is padded with EOS or with id 0 (transformers' pooling for the
        published `eos_token_id: 2` configs, and the first-EOS pooling of newer ones, agree on such prompts)."""
        pooled = last[torch.arange(last.shape[0], device=last.device), input_ids.to(last.device).argmax(-1)]
        g = self._proj_group()
        g.prepare()
        pack_lora([g], self.__dict__["_proj_jobs"])
        repack_trained([g], self.__dict__["_proj_repack"])
        return g([pooled.contiguous()]).float()

    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                output_hidden_states: bool = False, return_dict: bool = True, **kwargs):
        if attention_mask is not None:
            raise NotImplementedError("attention_mask on the text encoder is not supported (the reference's default "
                                      "use_attention_mask=False never passes one)")
        hs = self.run_layers(input_ids, len(self.text_model.encoder.layers), position_ids)
        last = self.final_norm(hs[-1])
        out = CLIPTextModelOutput(last_hidden_state=last, pooler_output=self.project(last, input_ids),
                                  hidden_states=tuple(hs) if output_hidden_states else None)
        return out if return_dict else out[:]


def _encoder(spec, cls):
    if spec is None:
        return cls()
    return cls(**spec) if isinstance(spec, dict) else spec


class SDXLTextEncoder(nn.Module):
    """The reference's SDXLTextEncoder (hcpdiff/models/compose/sdxl_composer.py, a ComposeTextEncoder): `clip_B` (CLIP ViT-L/14, the
    SD1.x encoder) and `clip_bigG` (CLIPTextModelWithProjection).  The submodule names are the reference's, so `re:.*self_attn$`
    selects the layers of both encoders, `re:clip_bigG.*` those of one, and checkpoint keys read
    `clip_B.text_model.encoder.layers.0.self_attn.q_proj.___.layer.W_down`.  Each argument is a module, a dict of its constructor
    keys, or None for the full-size encoder.  Run through `encode_prompt_sdxl`."""

    def __init__(self, clip_B=None, clip_bigG=None):
        super().__init__()
        self.clip_B = _encoder(clip_B, CLIPTextModel)
        self.clip_bigG = _encoder(clip_bigG, CLIPTextModelWithProjection)
        if not isinstance(self.clip_bigG, CLIPTextModelWithProjection):
            raise TypeError("clip_bigG must be a CLIPTextModelWithProjection (its projected pooled row is SDXL's text_embeds)")

    @property
    def dtype(self) -> torch.dtype:
        return self.clip_B.dtype

    @property
    def device(self) -> torch.device:
        return self.clip_B.device

    def linear_groups(self) -> List[LinearGroup]:
        return self.clip_B.linear_groups() + self.clip_bigG.linear_groups()

    def forward(self, input_ids: torch.Tensor, **kwargs):
        """(ehs, text_embeds) with all layers and the final norm (encode_prompt_sdxl with clip_skip 0)."""
        return encode_prompt_sdxl(self, input_ids)


def encode_prompt_sdxl(te: SDXLTextEncoder, input_ids: torch.Tensor, clip_skip: int = 0,
                       clip_final_norm: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's SDXL prompt path (ComposeTextEncoder with a TEEXHook per encoder, compose_textencoder.py:83-99, and
    SDXLTEUnetWrapper.forward, wrapper.py:57-75): ids [B, 2 x 77] are split in halves, the first for clip_B and the second for
    clip_bigG; each half gives the hidden state `clip_skip` layers before its last (final LayerNorm when `clip_final_norm`), and
    the two are concatenated on the channel axis -> ehs bf16 [B, 77, C_B + C_G].  `text_embeds` fp32 [B, projection_dim] is
    clip_bigG's text_projection(final_layer_norm(last layer)[row of the largest id]): all of bigG's layers run whatever
    `clip_skip` is, so with clip_skip > 0 its last layer is trained through text_embeds only.  clip_B runs only the layers it
    needs; its pooled output is discarded by the reference.  One 77-token chunk per encoder (n_repeats 1)."""
    B, L2 = input_ids.shape
    if L2 % 2:
        raise ValueError(f"input_ids width {L2}: SDXL ids are [batch, 2 x tokens] (clip_B's half, then clip_bigG's)")
    ids_b, ids_g = input_ids.chunk(2, -1)
    ehs_b = encode_prompt(te.clip_B, ids_b, 1, clip_skip, clip_final_norm)
    g = te.clip_bigG
    n_g = len(g.text_model.encoder.layers)
    if not 0 <= clip_skip < n_g:
        raise ValueError(f"clip_skip must be in [0, {n_g})")
    ids_g = ids_g.contiguous()
    hs = g.run_layers(ids_g, n_g)
    last = g.final_norm(hs[-1])
    if clip_skip == 0 and clip_final_norm:
        ehs_g = last
    else:
        ehs_g = _compose(g, hs[n_g - clip_skip], B, 1, clip_final_norm)
    text_embeds = g.project(last, ids_g)
    return torch.cat([ehs_b, ehs_g], dim=-1), text_embeds
