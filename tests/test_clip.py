"""CPU tests of the text-encoder surface: the module tree against the reference's cfgs/te_struct.txt, LoRA selection by the
reference's `lora_text_encoder` regexes, checkpoint / webui key schemes, and the fp32 restatement (tests/clip_ref.py) against vectors
of the real transformers CLIPTextModel + TEEXHook (tests/golden/ref_clip_text.pt)."""
import json
import os

import pytest
import torch

import clip_ref as R
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: F401  (models before runtime users)
from hcp_diffusion_b200.models.lora import LoraLayer
from hcp_diffusion_b200.tools.lora_convert import LoraConverter
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff

TE_ITEM = {"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}     # lora_conventional.yaml's lora_text_encoder


def test_clip_l_structure_matches_reference_dump(golden_dir):
    ref = json.load(open(os.path.join(golden_dir, "te_struct_clip_l.json")))
    te = CLIPTextModel()
    got = [[n, list(p.shape)] for n, p in te.named_parameters()]
    assert sorted(got) == sorted(ref)
    assert sum(p.numel() for p in te.parameters()) == 123_060_480
    assert te.text_model.encoder.layers[0].layer_norm1.eps == 1e-5
    # the oracle's parameter list is the same tree
    assert {n: tuple(s) for n, s in ref} == R.param_shapes(R.CLIP_L)


def test_transformers_state_dict_loads_strictly():
    transformers = pytest.importorskip("transformers")
    spec = R.SMALL
    cfg = transformers.CLIPTextConfig(**spec.kwargs(), hidden_act="quick_gelu")
    sd = {k: v for k, v in transformers.CLIPTextModel(cfg).state_dict().items() if "position_ids" not in k}
    CLIPTextModel(**spec.kwargs()).load_state_dict(sd, strict=True)


def test_lora_text_encoder_item_wraps_72_linears():
    te = CLIPTextModel().requires_grad_(False)
    _, group = make_hcpdiff(te, None, [TE_ITEM])
    blocks = group.plugin_dict
    assert len(blocks) == 72
    assert sorted(blocks) == sorted(R.lora_target_layers(R.CLIP_L))
    assert all(isinstance(b, LoraLayer) and b.rank == 4 for b in blocks.values())
    assert sum(p.numel() for b in blocks.values() for p in b.parameters()) == 663_552


def test_unsupported_options_raise():
    with pytest.raises(NotImplementedError):
        CLIPTextModel(hidden_act="gelu")
    te = CLIPTextModel(**R.SMALL.kwargs())
    with pytest.raises(NotImplementedError, match="attention_mask"):
        te(torch.zeros(1, 77, dtype=torch.long), attention_mask=torch.ones(1, 77))


def test_checkpoint_and_webui_keys_round_trip():
    te = CLIPTextModel(**R.SMALL.kwargs()).requires_grad_(False)
    _, group = make_hcpdiff(te, None, [TE_ITEM])
    with torch.no_grad():
        for b in group.plugin_dict.values():
            b.layer.W_up.normal_()
    sd = group.state_dict()
    assert "text_model.encoder.layers.0.self_attn.q_proj.___.layer.W_down" in sd
    assert "text_model.encoder.layers.2.mlp.fc2.___.layer.W_up" in sd
    web = LoraConverter().convert_to_webui({}, sd)
    assert "lora_te_text_model_encoder_layers_0_self_attn_q_proj.lora_down.weight" in web
    assert "lora_te_text_model_encoder_layers_1_mlp_fc1.lora_up.weight" in web
    back_te, back_unet = LoraConverter().convert_from_webui(web)
    assert not back_unet.get("lora")
    back = back_te["lora"]
    assert sorted(back) == sorted(sd)
    for k, v in sd.items():
        assert torch.equal(back[k], v), k


def test_oracle_matches_transformers_and_teexhook_golden(golden_dir):
    g = torch.load(os.path.join(golden_dir, "ref_clip_text.pt"))
    spec = R.SMALL
    sd = R.init_params(spec, R.GOLDEN_SEED)
    hs = R.hidden_states(sd, g["plain"]["ids"], spec)
    assert len(hs) == len(g["plain"]["hidden_states"]) == spec.num_hidden_layers + 1
    for i, (a, b) in enumerate(zip(hs, g["plain"]["hidden_states"])):
        err = float((a - b).norm() / b.norm())
        assert err < 1e-5, (i, err)
    last = R.final_norm(sd, hs[-1], spec)
    assert float((last - g["plain"]["last_hidden_state"]).norm() / last.norm()) < 1e-5
    assert len(g["cases"]) == len(R.GOLDEN_CASES)
    for c in g["cases"]:
        got = R.encode_prompt(sd, c["ids"], spec, c["n_repeats"], c["clip_skip"], c["clip_final_norm"])
        assert got.shape == c["ehs"].shape == (c["ids"].shape[0], 75 * c["n_repeats"] + 2, spec.hidden_size)
        err = float((got - c["ehs"]).norm() / c["ehs"].norm())
        assert err < 1e-5, (c["clip_skip"], c["clip_final_norm"], c["n_repeats"], err)


@pytest.mark.parametrize("extra,match", [
    ("text_encoder:\n  - {lr: 1e-6, layers: ['re:.*mlp$']}\n", "text_encoder:"),
    ("tokenizer_pt:\n  train:\n    - {name: pt-cat, lr: 3e-3}\n", "tokenizer_pt.train"),
    ("lora_text_encoder:\n  - {type: dapp, rank: 4, layers: ['re:.*mlp$']}\n", "DreamArtist"),
])
def test_train_ac_refuses_text_encoder_options_it_does_not_train(tmp_path, extra, match):
    from types import SimpleNamespace

    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    path = os.path.join(tmp_path, "c.yaml")
    with open(path, "w") as f:
        f.write("model: {clip_skip: 0}\n" + extra)
    with pytest.raises(NotImplementedError, match=match):
        Trainer._build_text_encoder(SimpleNamespace(device="cpu"), load_config_with_cli(path, args_list=[]))


def test_lora_te_config_mirrors_lora_conventional():
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    c = load_config_with_cli(os.path.join(root, "cfgs/train/lora_te_sd15_synthetic.yaml"), args_list=[])
    (item,) = c.lora_text_encoder
    assert float(item["lr"]) == 1e-5 and item["rank"] == 4 and list(item["layers"]) == ["re:.*self_attn$", "re:.*mlp$"]
    assert c.lora_unet[0]["rank"] == 8 and list(c.lora_unet[0]["layers"]) == [r"re:.*\.attn.?$", r"re:.*\.ff$"]
    assert c.model.clip_skip == 0 and c.model.clip_final_norm is True and c.model.tokenizer_repeats == 1
