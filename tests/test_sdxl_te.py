"""CPU tests of SDXL's text-encoder pair: the fp32 restatement (tests/sdxl_te_ref.py) against vectors of the real transformers models +
the reference's SDXLTextEncoder / TEEXHook (tests/golden/ref_sdxl_te.pt), the full-size OpenCLIP-bigG module tree against
transformers' CLIPTextModelWithProjection built from the published stable-diffusion-xl-base-1.0 `text_encoder_2` config, LoRA
selection by the reference's regexes, the training config and the refusals."""
import os
from types import SimpleNamespace

import pytest
import torch

import sdxl_te_ref as X
from hcp_diffusion_b200.models import CLIPTextModel, CLIPTextModelWithProjection, SDXLTextEncoder, UNet2DConditionModel
from hcp_diffusion_b200.models.lora import LoraLayer
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff
from oracle import unet_ref as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TE_ITEM = {"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}        # lora_sdxl.yaml's lora_text_encoder item
# stable-diffusion-xl-base-1.0/text_encoder_2/config.json (OpenCLIP ViT-bigG/14)
BIGG_CONFIG = dict(vocab_size=49408, hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=20,
                   max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5, projection_dim=1280, bos_token_id=0, eos_token_id=2,
                   pad_token_id=1)


def test_restatement_matches_reference_golden(golden_dir):
    g = torch.load(os.path.join(golden_dir, "ref_sdxl_te.pt"))
    pair = X.TINY_XL_TE
    sd = X.init_params(pair, X.GOLDEN_SEED)
    assert len(g["cases"]) == len(X.GOLDEN_CASES)
    assert {(c["clip_skip"], c["clip_final_norm"], c["pad_g"]) for c in g["cases"]} == set(X.GOLDEN_CASES)
    for c in g["cases"]:
        ids = c["ids"]
        # the layouts: clip_B's chunk padded with EOS; bigG's chunk with the case's padding after its one EOS
        assert ids.shape == (2, 154) and bool((ids[:, 76] == X.EOS).all()) and bool((ids[:, 153] == c["pad_g"]).all())
        # the pooled row does not depend on the configs' eos_token_id (2: argmax of the ids; 49407: first EOS)
        torch.testing.assert_close(c["text_embeds_eos49407"], c["text_embeds"], rtol=0, atol=0)
        ehs, te = X.encode_prompt_sdxl(sd, ids, pair, c["clip_skip"], c["clip_final_norm"])
        assert ehs.shape == c["ehs"].shape == (2, 77, 64) and te.shape == c["text_embeds"].shape == (2, 64)
        for got, want in ((ehs, c["ehs"]), (te, c["text_embeds"])):
            err = float((got - want).norm() / want.norm())
            assert err < 1e-5, (c["clip_skip"], c["clip_final_norm"], c["pad_g"], err)


def test_full_size_bigg_matches_transformers_tree():
    transformers = pytest.importorskip("transformers")
    with torch.device("meta"):
        ref = transformers.CLIPTextModelWithProjection(transformers.CLIPTextConfig(**BIGG_CONFIG))
        ours = CLIPTextModelWithProjection()
    want = {n: tuple(p.shape) for n, p in ref.named_parameters()}
    got = {n: tuple(p.shape) for n, p in ours.named_parameters()}
    assert got == want
    assert sum(p.numel() for p in ours.parameters()) == 694_659_840
    assert got == {k[len("clip_bigG."):]: v for k, v in X.param_shapes(X.FULL).items() if k.startswith("clip_bigG.")}
    assert type(ours.text_model.encoder.layers[0].mlp.activation_fn).__name__ == "GELUActivation"
    assert ours.text_projection.bias is None


def test_transformers_state_dicts_load_strictly():
    transformers = pytest.importorskip("transformers")
    pair = X.SMALL_XL
    g = transformers.CLIPTextModelWithProjection(transformers.CLIPTextConfig(**pair.clip_bigG.kwargs(), hidden_act="gelu",
                                                                             projection_dim=pair.projection_dim))
    b = transformers.CLIPTextModel(transformers.CLIPTextConfig(**pair.clip_B.kwargs(), hidden_act="quick_gelu"))
    te = SDXLTextEncoder(**pair.kwargs())
    sd = {f"clip_B.{k}": v for k, v in b.state_dict().items() if "position_ids" not in k}
    sd.update({f"clip_bigG.{k}": v for k, v in g.state_dict().items() if "position_ids" not in k})
    te.load_state_dict(sd, strict=True)
    assert {n: tuple(p.shape) for n, p in te.named_parameters()} == X.param_shapes(pair)


def test_sd1_encoder_still_refuses_exact_gelu():
    with pytest.raises(NotImplementedError, match="CLIPTextModelWithProjection"):
        CLIPTextModel(hidden_act="gelu")
    with pytest.raises(NotImplementedError):
        CLIPTextModelWithProjection(hidden_act="relu")
    with pytest.raises(TypeError, match="clip_bigG"):
        SDXLTextEncoder(clip_B=X.TINY_XL_TE.clip_B.kwargs(), clip_bigG=CLIPTextModel(**X.TINY_XL_TE.clip_bigG.kwargs()))


def test_lora_items_select_both_or_one_encoder():
    with torch.device("meta"):
        te = SDXLTextEncoder().requires_grad_(False)
    _, group = make_hcpdiff(te, None, [dict(TE_ITEM)])
    blocks = group.plugin_dict
    assert len(blocks) == 72 + 192
    assert sorted(blocks) == sorted(X.lora_target_layers(X.FULL))
    assert all(isinstance(b, LoraLayer) and b.rank == 4 for b in blocks.values())
    te = SDXLTextEncoder(**X.TINY_XL_TE.kwargs()).requires_grad_(False)
    _, group = make_hcpdiff(te, None, [{"rank": 4, "layers": [r"re:clip_bigG.*self_attn$", r"re:clip_bigG.*mlp$"]}])
    assert sorted(group.plugin_dict) == sorted(n for n in X.lora_target_layers(X.TINY_XL_TE) if n.startswith("clip_bigG."))
    assert "clip_bigG.text_model.encoder.layers.0.self_attn.q_proj.___.layer.W_down" in group.state_dict()


def test_synthetic_ids_layout():
    ids = X.synthetic_ids(3, seed=5)
    b, g = ids[:, :77], ids[:, 77:]
    assert bool((b[:, 0] == X.BOS).all()) and bool((g[:, 0] == X.BOS).all())
    for r in range(3):
        n = int((b[r] != X.EOS).sum()) - 1                       # words after BOS
        assert torch.equal(b[r, :n + 1], g[r, :n + 1]) and int(g[r, n + 1]) == X.EOS
        assert bool((b[r, n + 1:] == X.EOS).all()) and bool((g[r, n + 2:] == 0).all())
        assert int(b[r].argmax()) == int(g[r].argmax()) == n + 1


def test_sdxl_te_config_mirrors_lora_sdxl():
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    c = load_config_with_cli(os.path.join(ROOT, "cfgs/train/lora_sdxl_te_synthetic.yaml"), args_list=[])
    (item,) = c.lora_text_encoder
    assert float(item["lr"]) == 1e-5 and item["rank"] == 4 and list(item["layers"]) == ["re:.*self_attn$", "re:.*mlp$"]
    (uitem,) = c.lora_unet
    assert float(uitem["lr"]) == 1e-4 and uitem["rank"] == 8 and list(uitem["layers"]) == [r"re:.*\.attn.?$", r"re:.*\.ff$"]
    assert c.model.clip_skip == 1 and c.model.clip_final_norm is False and c.model.tokenizer_repeats == 1
    assert c.model.unet.addition_embed_type == "text_time" and c.model.unet.cross_attention_dim == 2048
    assert "text_encoder" not in c.model                    # the SDXL pair is the default for a text_time UNet


def tiny_xl_unet():
    spec = U.TINY_XL
    u = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
                             cross_attention_dim=spec.cross_attention_dim, down_block_types=["DownBlock2D", "CrossAttnDownBlock2D",
                                                                                              "CrossAttnDownBlock2D"],
                             up_block_types=["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"],
                             transformer_layers_per_block=spec.transformer_depth, use_linear_projection=True,
                             addition_embed_type="text_time", addition_time_embed_dim=spec.addition_time_embed_dim,
                             projection_class_embeddings_input_dim=spec.projection_class_embeddings_input_dim)
    return u.requires_grad_(False)


def test_engine_refusals():
    from hcp_diffusion_b200.engine import LoraTrainStep
    unet = tiny_xl_unet()
    groups, _ = make_hcpdiff(unet, None, [{"rank": 4, "layers": [r"re:.*\.attn.?$"]}])
    te = SDXLTextEncoder(**X.TINY_XL_TE.kwargs()).requires_grad_(False)
    tgroups, _ = make_hcpdiff(te, None, [dict(TE_ITEM)])
    with pytest.raises(NotImplementedError, match="raw tokenizer output"):
        LoraTrainStep(unet, groups + tgroups, text_encoder=te, text_encoder_opts={"n_repeats": 2}, use_cuda_graph=False)
    with pytest.raises(NotImplementedError, match="cfg_scale"):
        LoraTrainStep(unet, groups + tgroups, text_encoder=te, cfg_scale="0.5-1.0")
    sd1 = CLIPTextModel(**X.TINY_XL_TE.clip_B.kwargs()).requires_grad_(False)
    sgroups, _ = make_hcpdiff(sd1, None, [dict(TE_ITEM)])
    with pytest.raises(NotImplementedError, match="SDXLTextEncoder"):
        LoraTrainStep(unet, groups + sgroups, text_encoder=sd1)
    step = LoraTrainStep(unet, groups + tgroups, text_encoder=te, text_encoder_opts={"clip_skip": 1}, use_cuda_graph=False)
    spec = U.TINY_XL
    lat, noise, t, _ = U.synthetic_batch(2, spec)
    ids = X.synthetic_ids(2)
    with pytest.raises(ValueError, match="text_embeds is computed"):
        step.step(lat, noise, t, ids, {"time_ids": torch.zeros(2, 6), "text_embeds": torch.zeros(2, 64)})
    with pytest.raises(ValueError, match="time_ids"):
        step.step(lat, noise, t, ids, None)
    # step_groups() checks every group the same way, before anything runs
    good = {"latents": lat, "noise": noise, "t": t, "ehs": ids, "added_cond_kwargs": {"time_ids": torch.zeros(2, 6)}}
    with pytest.raises(ValueError, match="group 1: .*time_ids"):
        step.step_groups([good, {k: v for k, v in good.items() if k != "added_cond_kwargs"}])
    with pytest.raises(ValueError, match="group 1: text_embeds is computed"):
        step.step_groups([good, dict(good, added_cond_kwargs={"time_ids": torch.zeros(2, 6), "text_embeds": torch.zeros(2, 64)})])


def test_train_ac_builds_the_sdxl_pair_for_a_text_time_unet(tmp_path):
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    path = os.path.join(tmp_path, "c.yaml")
    with open(path, "w") as f:
        f.write("model: {clip_skip: 1, clip_final_norm: false}\nlora_text_encoder:\n  - {rank: 4, layers: ['re:.*self_attn$']}\n")
    cfg = load_config_with_cli(path, args_list=[])
    unet = SimpleNamespace(config=SimpleNamespace(addition_embed_type="text_time"))
    with torch.device("meta"):
        te, _, opts = Trainer._build_text_encoder(SimpleNamespace(device="meta", unet=unet), cfg)
    assert isinstance(te, SDXLTextEncoder) and sum(p.numel() for p in te.clip_bigG.parameters()) == 694_659_840
    assert opts == {"n_repeats": 1, "clip_skip": 1, "clip_final_norm": False}
    unet.config.addition_embed_type = None
    with torch.device("meta"):
        te, _, _ = Trainer._build_text_encoder(SimpleNamespace(device="meta", unet=unet), cfg)
    assert type(te) is CLIPTextModel
