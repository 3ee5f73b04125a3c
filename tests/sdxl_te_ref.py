"""fp32 CPU restatement of SDXL's text-encoder pair with the reference's LoRA operator: transformers' CLIPTextModel (`clip_B`) and
CLIPTextModelWithProjection (`clip_bigG`, exact-GELU MLP, bias-free `text_projection`), composed as the reference's SDXLTextEncoder
with a TEEXHook per encoder (hcpdiff/models/compose/compose_textencoder.py:83-99, textencoder_ex.py:65-82) and read as
SDXLTEUnetWrapper does (wrapper.py:57-75: text_embeds = bigG's pooled output).  Test infrastructure only; pinned to the real
transformers models + the reference's classes by tests/golden/ref_sdxl_te.pt (tests/golden/make_golden_sdxl_te.py).
"""
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

import clip_ref as R
from oracle.unet_ref import LoraEntry, _linear

BOS, EOS, PAD_G = R.BOS, R.EOS, 0          # SDXL's second tokenizer pads with '!' (id 0) after EOS; the first pads with EOS


@dataclass(frozen=True)
class PairSpec:
    clip_B: R.CLIPSpec
    clip_bigG: R.CLIPSpec
    projection_dim: int

    def kwargs(self) -> dict:
        """SDXLTextEncoder constructor keys."""
        return {"clip_B": self.clip_B.kwargs(), "clip_bigG": {**self.clip_bigG.kwargs(), "projection_dim": self.projection_dim}}


CLIP_BIGG = R.CLIPSpec(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=20)
FULL = PairSpec(R.CLIP_L, CLIP_BIGG, 1280)
# sized to oracle.unet_ref.TINY_XL: context 32 + 32 = 64 channels, text_embeds 256 - 6 x 32 = 64
TINY_XL_TE = PairSpec(R.CLIPSpec(hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=1),
                      R.CLIPSpec(hidden_size=32, intermediate_size=64, num_hidden_layers=3, num_attention_heads=1), 64)
# head dim 64 as in the full-size pair
SMALL_XL = PairSpec(R.SMALL, R.CLIPSpec(hidden_size=128, intermediate_size=512, num_hidden_layers=4, num_attention_heads=2), 96)


def _prefixed(d: dict, prefix: str) -> dict:
    return {prefix + k: v for k, v in d.items()}


def param_shapes(pair: PairSpec) -> Dict[str, tuple]:
    out = _prefixed(R.param_shapes(pair.clip_B), "clip_B.")
    out.update(_prefixed(R.param_shapes(pair.clip_bigG), "clip_bigG."))
    out["clip_bigG.text_projection.weight"] = (pair.projection_dim, pair.clip_bigG.hidden_size)
    return out


def init_params(pair: PairSpec, seed: int = 0) -> Dict[str, Tensor]:
    sd = _prefixed(R.init_params(pair.clip_B, seed), "clip_B.")
    sd.update(_prefixed(R.init_params(pair.clip_bigG, seed + 1), "clip_bigG."))
    g = torch.Generator().manual_seed(seed + 2)
    C_ = pair.clip_bigG.hidden_size
    sd["clip_bigG.text_projection.weight"] = torch.randn((pair.projection_dim, C_), generator=g) / math.sqrt(C_)
    return sd


def lora_target_layers(pair: PairSpec) -> List[str]:
    """Layers `re:.*self_attn$` and `re:.*mlp$` wrap in both encoders (reference lora_sdxl.yaml's lora_text_encoder item)."""
    return [f"clip_B.{n}" for n in R.lora_target_layers(pair.clip_B)] + [f"clip_bigG.{n}" for n in R.lora_target_layers(pair.clip_bigG)]


def init_lora(pair: PairSpec, rank: int = 4, seed: int = 2, up_std: float = 0.02) -> Dict[str, List[LoraEntry]]:
    out = _prefixed(R.init_lora(pair.clip_B, rank, seed=seed, up_std=up_std), "clip_B.")
    out.update(_prefixed(R.init_lora(pair.clip_bigG, rank, seed=seed + 1, up_std=up_std), "clip_bigG."))
    return out


def synthetic_ids(batch: int, seed: int = 7, n_words=None, pad_g: int = PAD_G) -> Tensor:
    """int64 [batch, 2 x 77]: clip_B's chunk (BOS, words, EOS padding), then bigG's with the same words, EOS, and `pad_g` padding."""
    ids_b = R.synthetic_ids(batch, 1, seed=seed, n_words=n_words)
    ids_g = ids_b.clone()
    for r in range(batch):
        first_eos = int((ids_b[r] == EOS).nonzero()[0])
        ids_g[r, first_eos + 1:] = pad_g
    return torch.cat([ids_b, ids_g], 1)


def hidden_states(sd: Dict[str, Tensor], prefix: str, ids: Tensor, spec: R.CLIPSpec, act: str, lora=None,
                  n_layers: Optional[int] = None) -> List[Tensor]:
    """clip_ref.hidden_states with the MLP activation as a parameter: 'quick_gelu' (CLIP-L) or 'gelu' (exact, OpenCLIP-bigG)."""
    B, L = ids.shape
    p0 = prefix + "text_model."
    h = sd[p0 + "embeddings.token_embedding.weight"][ids] + sd[p0 + "embeddings.position_embedding.weight"][:L]
    H, C_ = spec.num_attention_heads, spec.hidden_size
    d = C_ // H
    mask = torch.full((L, L), float("-inf"), device=h.device).triu(1)
    out = [h]
    for i in range(spec.num_hidden_layers if n_layers is None else n_layers):
        p = f"{p0}encoder.layers.{i}."
        x = R._layer_norm(sd, p + "layer_norm1", h, spec.layer_norm_eps)
        q, k, v = (_linear(sd, lora, p + f"self_attn.{n}", x).view(B, L, H, d).transpose(1, 2) for n in ("q_proj", "k_proj", "v_proj"))
        a = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5 + mask, -1) @ v
        h = h + _linear(sd, lora, p + "self_attn.out_proj", a.transpose(1, 2).reshape(B, L, C_))
        x = R._layer_norm(sd, p + "layer_norm2", h, spec.layer_norm_eps)
        u = _linear(sd, lora, p + "mlp.fc1", x)
        u = u * torch.sigmoid(1.702 * u) if act == "quick_gelu" else torch.nn.functional.gelu(u)
        h = h + _linear(sd, lora, p + "mlp.fc2", u)
        out.append(h)
    return out


def final_norm(sd, prefix: str, h: Tensor, spec: R.CLIPSpec) -> Tensor:
    return R._layer_norm(sd, prefix + "text_model.final_layer_norm", h, spec.layer_norm_eps)


def encode_prompt_sdxl(sd: Dict[str, Tensor], ids: Tensor, pair: PairSpec, clip_skip: int = 0, clip_final_norm: bool = True, lora=None,
                       training: bool = False) -> Tuple[Tensor, Tensor]:
    """-> (ehs [B, 77, C_B + C_G], text_embeds [B, projection_dim]).  Per encoder: hidden_states[-clip_skip - 1], final LayerNorm when
    `clip_final_norm` (and, with `training` and clip_skip > 0, + 0 * last_hidden_state.mean() as TEEXHook does).  text_embeds =
    text_projection(final_layer_norm(bigG's last layer)[row of the largest id]) (transformers' pooling for eos_token_id 2)."""
    ids_b, ids_g = ids.chunk(2, -1)
    outs = []
    for prefix, spec, act, part in (("clip_B.", pair.clip_B, "quick_gelu", ids_b), ("clip_bigG.", pair.clip_bigG, "gelu", ids_g)):
        hs = hidden_states(sd, prefix, part, spec, act, lora)
        h = hs[spec.num_hidden_layers - clip_skip]
        if clip_final_norm:
            h = final_norm(sd, prefix, h, spec)
        last = final_norm(sd, prefix, hs[-1], spec)
        if training and clip_skip > 0:
            h = h + 0 * last.mean()
        outs.append((h, last))
    (ehs_b, _), (ehs_g, last_g) = outs
    pooled = last_g[torch.arange(ids.shape[0]), ids_g.argmax(-1)]
    text_embeds = _linear(sd, lora, "clip_bigG.text_projection", pooled)
    return torch.cat([ehs_b, ehs_g], -1), text_embeds


# golden cases of tests/golden/ref_sdxl_te.pt: (clip_skip, clip_final_norm) x bigG padding (0: SDXL's tokenizer_2, EOS: as tokenizer)
GOLDEN_CASES = [(s, f, pad) for s in (0, 1) for f in (True, False) for pad in (PAD_G, EOS)]
GOLDEN_SEED = 13


def joint_reference_loop(unet_sd, unet_lora, unet_spec, te_sd, te_lora, pair, clip_skip, clip_final_norm, lr=1e-4, te_lr=1e-5,
                         optimizer_kwargs=None, **kw):
    """oracle.step_ref.ReferenceLoop with SDXL's pair in front (SDXLTEUnetWrapper.forward): ehs and text_embeds from the encoders, the
    text-encoder adapters one more parameter group under the shared global-norm clip; AdamW, or with `optimizer_kwargs` Adafactor
    (tests/adafactor_ref.py).  `micro_step(latents, noise, t, ids, time_ids)`."""
    from oracle import step_ref as S

    class Joint(S.ReferenceLoop):
        def __init__(self):
            super().__init__(unet_sd, unet_lora, unet_spec, lr=lr, **kw)
            leaves = [p for blocks in te_lora.values() for e in blocks for p in (e.W_down, e.W_up)]
            for p in leaves:
                p.requires_grad_(True)
            self.opt.add_param_group({"params": leaves, "lr": te_lr})
            self.leaves += leaves
            if optimizer_kwargs is not None:
                import adafactor_ref as A
                opts = dict(optimizer_kwargs)
                opts.pop("lr", None)
                self.opt = A.OracleAdafactor([{"params": g["params"], "lr": g["lr"]} for g in self.opt.param_groups], **opts)

        def micro_step(self, latents, noise, t, ids, time_ids):
            ehs, text_embeds = encode_prompt_sdxl(te_sd, ids, pair, clip_skip, clip_final_norm, lora=te_lora, training=True)
            return super().micro_step(latents, noise, t, ehs, added_cond_kwargs={"text_embeds": text_embeds, "time_ids": time_ids})

    return Joint()
