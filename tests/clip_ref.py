"""fp32 CPU restatement of transformers' CLIPTextModel (the SD1.x text encoder) with the reference's LoRA operator, and of the
reference's prompt composition (hcpdiff/models/textencoder_ex.py TEEXHook: split into 77-token chunks, clip_skip, final norm,
BOS + middle rows + EOS).  Test infrastructure only; pinned to the real transformers model and TEEXHook by
tests/golden/ref_clip_text.pt (tests/golden/make_golden_clip.py).
"""
import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
from torch import Tensor

from oracle.unet_ref import LoraEntry, _linear

BOS, EOS = 49406, 49407


@dataclass(frozen=True)
class CLIPSpec:
    vocab_size: int = 49408
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    max_position_embeddings: int = 77
    layer_norm_eps: float = 1e-5

    def kwargs(self) -> dict:
        return dict(vocab_size=self.vocab_size, hidden_size=self.hidden_size, intermediate_size=self.intermediate_size,
                    num_hidden_layers=self.num_hidden_layers, num_attention_heads=self.num_attention_heads,
                    max_position_embeddings=self.max_position_embeddings, layer_norm_eps=self.layer_norm_eps)


CLIP_L = CLIPSpec()
# the text encoder of the TINY UNet (cross_attention_dim 64): one head of 64
TINY_TE = CLIPSpec(hidden_size=64, intermediate_size=256, num_hidden_layers=2, num_attention_heads=1)
# a small encoder with the real vocabulary and context length (BOS / EOS ids are the tokenizer's): head dim 64 like CLIP-L
SMALL = CLIPSpec(hidden_size=128, intermediate_size=512, num_hidden_layers=3, num_attention_heads=2)


def param_shapes(spec: CLIPSpec) -> Dict[str, tuple]:
    C_, F_ = spec.hidden_size, spec.intermediate_size
    out = {"text_model.embeddings.token_embedding.weight": (spec.vocab_size, C_),
           "text_model.embeddings.position_embedding.weight": (spec.max_position_embeddings, C_)}
    for i in range(spec.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            out[p + f"self_attn.{n}.weight"], out[p + f"self_attn.{n}.bias"] = (C_, C_), (C_,)
        out[p + "layer_norm1.weight"], out[p + "layer_norm1.bias"] = (C_,), (C_,)
        out[p + "mlp.fc1.weight"], out[p + "mlp.fc1.bias"] = (F_, C_), (F_,)
        out[p + "mlp.fc2.weight"], out[p + "mlp.fc2.bias"] = (C_, F_), (C_,)
        out[p + "layer_norm2.weight"], out[p + "layer_norm2.bias"] = (C_,), (C_,)
    out["text_model.final_layer_norm.weight"], out["text_model.final_layer_norm.bias"] = (C_,), (C_,)
    return out


def init_params(spec: CLIPSpec, seed: int = 0) -> Dict[str, Tensor]:
    """Seeded weights with CLIP-like scales: N(0, 0.02) embeddings, linears at 1/sqrt(fan_in), LayerNorm affine near (1, 0)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shp in param_shapes(spec).items():
        if "embedding" in name:
            t = torch.randn(shp, generator=g) * 0.02
        elif "norm" in name:
            t = (1.0 if name.endswith("weight") else 0.0) + torch.randn(shp, generator=g) * 0.05
        elif name.endswith("weight"):
            t = torch.randn(shp, generator=g) / math.sqrt(shp[1])
        else:
            t = torch.randn(shp, generator=g) * 0.02
        sd[name] = t
    return sd


def lora_target_layers(spec: CLIPSpec) -> List[str]:
    """Layers `re:.*self_attn$` and `re:.*mlp$` wrap (reference lora_conventional.yaml's lora_text_encoder item)."""
    out = []
    for i in range(spec.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}."
        out += [p + f"self_attn.{n}" for n in ("k_proj", "v_proj", "q_proj", "out_proj")] + [p + "mlp.fc1", p + "mlp.fc2"]
    return out


def init_lora(spec: CLIPSpec, rank: int = 4, alpha: float = 1.0, seed: int = 2, up_std: float = 0.02) -> Dict[str, List[LoraEntry]]:
    shapes = param_shapes(spec)
    out = {}
    for idx, layer in enumerate(lora_target_layers(spec)):
        o, i = shapes[layer + ".weight"]
        g = torch.Generator().manual_seed(seed * 7_000_003 + idx)
        down = (torch.rand((rank, i), generator=g) * 2 - 1) / math.sqrt(i)
        up = torch.randn((o, rank), generator=g) * up_std
        out[layer] = [LoraEntry(down, up, alpha / rank, None)]
    return out


def synthetic_ids(batch: int, n_repeats: int = 1, seed: int = 7, n_words=None) -> Tensor:
    """int64 [batch, 77 R]: per chunk BOS, `n_words` random tokens, then EOS padding (the SD1.x tokenizer's pad token)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((batch * n_repeats, 77), EOS, dtype=torch.int64)
    ids[:, 0] = BOS
    for r in range(batch * n_repeats):
        n = int(torch.randint(5, 70, (1,), generator=g)) if n_words is None else n_words
        ids[r, 1:1 + n] = torch.randint(0, 49406, (n,), generator=g)
    return ids.reshape(batch, 77 * n_repeats)


def _layer_norm(sd, name, x, eps):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def hidden_states(sd: Dict[str, Tensor], ids: Tensor, spec: CLIPSpec, lora=None, n_layers: Optional[int] = None) -> List[Tensor]:
    """[embeddings, layer 1, ..., layer n] of CLIPTextTransformer (pre-LN layers, causal self-attention, quick-GELU MLP)."""
    B, L = ids.shape
    h = sd["text_model.embeddings.token_embedding.weight"][ids.to(sd["text_model.final_layer_norm.weight"].device)] + \
        sd["text_model.embeddings.position_embedding.weight"][:L]
    H, C_ = spec.num_attention_heads, spec.hidden_size
    d = C_ // H
    mask = torch.full((L, L), float("-inf"), device=h.device).triu(1)
    out = [h]
    for i in range(spec.num_hidden_layers if n_layers is None else n_layers):
        p = f"text_model.encoder.layers.{i}."
        x = _layer_norm(sd, p + "layer_norm1", h, spec.layer_norm_eps)
        q, k, v = (_linear(sd, lora, p + f"self_attn.{n}", x).view(B, L, H, d).transpose(1, 2) for n in ("q_proj", "k_proj", "v_proj"))
        a = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5 + mask, -1) @ v
        h = h + _linear(sd, lora, p + "self_attn.out_proj", a.transpose(1, 2).reshape(B, L, C_))
        x = _layer_norm(sd, p + "layer_norm2", h, spec.layer_norm_eps)
        u = _linear(sd, lora, p + "mlp.fc1", x)
        h = h + _linear(sd, lora, p + "mlp.fc2", u * torch.sigmoid(1.702 * u))
        out.append(h)
    return out


def final_norm(sd, h, spec: CLIPSpec) -> Tensor:
    return _layer_norm(sd, "text_model.final_layer_norm", h, spec.layer_norm_eps)


def encode_prompt(sd: Dict[str, Tensor], ids: Tensor, spec: CLIPSpec, n_repeats: int = 1, clip_skip: int = 0, clip_final_norm: bool = True,
                  lora=None, training: bool = False) -> Tensor:
    """TEEXHook.forward_hook_input + forward_hook (textencoder_ex.py:55-82) -> [B, 75 R + 2, C].  `training` with clip_skip > 0 adds
    0 * last_hidden_state.mean() as the reference does, so the adapters of the skipped layers get a zero gradient (and AdamW decay)."""
    B = ids.shape[0]
    hs = hidden_states(sd, ids.reshape(B * n_repeats, -1), spec, lora)
    h = hs[spec.num_hidden_layers - clip_skip]
    if clip_final_norm:
        h = final_norm(sd, h, spec)
    if training and clip_skip > 0:
        h = h + 0 * final_norm(sd, hs[-1], spec).mean()
    h = h.reshape(B, n_repeats, *h.shape[1:])
    return torch.cat([h[:, 0, :1], h[:, :, 1:-1].flatten(1, 2), h[:, -1, -1:]], dim=1)


# golden cases of tests/golden/ref_clip_text.pt: (clip_skip, clip_final_norm, n_repeats)
GOLDEN_CASES = [(s, f, r) for s in (0, 1) for f in (True, False) for r in (1, 2)]
GOLDEN_SEED = 11


def joint_reference_loop(unet_sd, unet_lora, unet_spec, te_sd, te_lora, te_spec, te_opts, lr=1e-4, te_lr=1e-5, **kw):
    """oracle.step_ref.ReferenceLoop with the text encoder in front (TEUnetWrapper.forward, hcpdiff/models/wrapper.py:14-30): the
    text-encoder adapters are one more AdamW group and share the global-norm clip; `micro_step` takes token ids."""
    from oracle import step_ref as S

    class Joint(S.ReferenceLoop):
        def __init__(self):
            super().__init__(unet_sd, unet_lora, unet_spec, lr=lr, **kw)
            leaves = [p for blocks in te_lora.values() for e in blocks for p in (e.W_down, e.W_up)]
            for p in leaves:
                p.requires_grad_(True)
            self.opt.add_param_group({"params": leaves, "lr": te_lr})
            self.leaves += leaves

        def micro_step(self, latents, noise, t, ids):
            ehs = encode_prompt(te_sd, ids, te_spec, lora=te_lora, training=True, **te_opts)
            return super().micro_step(latents, noise, t, ehs)

    return Joint()
