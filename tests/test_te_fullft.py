"""Full fine-tuning of the text encoder without a GPU: the `text_encoder:` config list, the refusals that remain, the saved 'base'
part of `text_encoder-<step>` (transformers' names, loadable into `transformers.CLIPTextModel`), the optimizer layouts for the
[vocab, C] token table and the new example config."""
import os
from types import SimpleNamespace

import pytest
import torch

import clip_ref as R
from hcp_diffusion_b200 import adafactor, adamw8bit
from hcp_diffusion_b200.ckpt_manager import CkptManagerPKL
from hcp_diffusion_b200.models import CLIPTextModel
from hcp_diffusion_b200.train_ac import Trainer
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff
from hcp_diffusion_b200.utils.config import load_config_with_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "cfgs", "train", "dreambooth_te_sd15_synthetic.yaml")


def tiny_te():
    te = CLIPTextModel(**R.TINY_TE.kwargs())
    te.load_state_dict(R.init_params(R.TINY_TE, seed=1))
    return te.requires_grad_(False)


def test_config_mirrors_fine_tuning_yaml_and_dreambooth():
    c = load_config_with_cli(CFG, args_list=[])
    (item,) = c.text_encoder
    assert float(item["lr"]) == 1e-6 and list(item["layers"]) == [""]
    (uitem,) = c.unet
    assert float(uitem["lr"]) == 1e-6 and list(uitem["layers"]) == [""]
    assert not c.get("lora_text_encoder") and not c.get("lora_unet")
    base = load_config_with_cli(os.path.join(ROOT, "cfgs/train/dreambooth_sd15_synthetic.yaml"), args_list=[])
    assert c.train.scheduler == base.train.scheduler and c.train.optimizer == base.train.optimizer
    assert set(c.data) == set(base.data)


def test_text_encoder_items_select_layers_with_default_lr():
    te = tiny_te()
    groups, lora = make_hcpdiff(te, [{"layers": ["text_model.encoder.layers.1", "text_model.embeddings"]},
                                     {"lr": 3e-6, "layers": ["re:.*final_layer_norm$"]}], None, default_lr=1e-5)
    assert lora.empty()
    assert [g["lr"] for g in groups] == [1e-5, 3e-6]
    names = {n for n, p in te.named_parameters() if p.requires_grad}
    assert names == {n for n in R.param_shapes(R.TINY_TE) if ".layers.1." in n or "embeddings" in n or "final_layer_norm" in n}
    assert sum(p.numel() for g in groups for p in g["params"]) == sum(p.numel() for n, p in te.named_parameters() if n in names)


def test_text_encoder_list_builds_the_encoder_without_lora_items(tmp_path):
    path = os.path.join(tmp_path, "c.yaml")
    with open(path, "w") as f:
        f.write("model:\n  clip_skip: 1\n  tokenizer_repeats: 2\n  text_encoder:\n    _target_: hcp_diffusion_b200.models.CLIPTextModel\n"
                "    hidden_size: 64\n    intermediate_size: 256\n    num_hidden_layers: 2\n    num_attention_heads: 1\n"
                "text_encoder:\n  - {lr: 1e-6, layers: ['']}\n")
    host = SimpleNamespace(device="meta", unet=SimpleNamespace(config=SimpleNamespace(addition_embed_type=None)))
    with torch.device("meta"):
        te, lora, opts = Trainer._build_text_encoder(host, load_config_with_cli(path, args_list=[]))
    assert isinstance(te, CLIPTextModel) and lora is None
    assert opts == {"n_repeats": 2, "clip_skip": 1, "clip_final_norm": True}
    assert not any(p.requires_grad for p in te.parameters())      # make_hcpdiff turns the selected layers on


@pytest.mark.parametrize("extra,match", [
    ("tokenizer_pt:\n  train:\n    - {name: pt-cat, lr: 3e-3}\n", "tokenizer_pt.train"),
    ("lora_text_encoder:\n  - {type: dapp, rank: 4, layers: ['re:.*mlp$']}\n", "DreamArtist"),
])
def test_remaining_refusals_with_a_text_encoder_list(tmp_path, extra, match):
    path = os.path.join(tmp_path, "c.yaml")
    with open(path, "w") as f:
        f.write("model: {clip_skip: 0}\ntext_encoder:\n  - {lr: 1e-6, layers: ['']}\n" + extra)
    with pytest.raises(NotImplementedError, match=match):
        Trainer._build_text_encoder(SimpleNamespace(device="cpu"), load_config_with_cli(path, args_list=[]))


@pytest.mark.parametrize("items", ["text_encoder:\n  - {lr: 1e-6, layers: ['re:.*mlp$']}\n",
                                   "lora_text_encoder:\n  - {rank: 4, layers: ['re:.*mlp$']}\n"])
def test_text_encoder_training_on_the_cpu_is_refused_before_building(tmp_path, items):
    """The text encoder has no CPU path: either list on a CPU device is refused before a full-size encoder is built."""
    path = os.path.join(tmp_path, "c.yaml")
    with open(path, "w") as f:
        f.write("model: {clip_skip: 0}\n" + items)
    with pytest.raises(NotImplementedError, match="CUDA"):
        Trainer._build_text_encoder(SimpleNamespace(device="cpu"), load_config_with_cli(path, args_list=[]))


def test_cfg_scale_with_a_fully_trained_text_encoder_is_refused():
    from hcp_diffusion_b200.engine import LoraTrainStep
    te = tiny_te()
    groups, _ = make_hcpdiff(te, [{"layers": [""]}], None)
    with pytest.raises(NotImplementedError, match="cfg_scale"):
        LoraTrainStep(torch.nn.Linear(2, 2), groups, cfg_scale="0.5-1.0", text_encoder=te)


def test_dapp_on_the_text_encoder_is_refused_at_run_time():
    te = tiny_te()
    make_hcpdiff(te, [{"layers": [""]}], [{"type": "dapp", "rank": 4, "layers": ["re:.*mlp$"]}])
    with pytest.raises(NotImplementedError, match="DreamArtist"):
        te._check_trainable()


def _saved_base(te, tmp_path):
    mgr = CkptManagerPKL()
    mgr.set_save_dir(str(tmp_path))
    path = mgr.save_model_with_lora(te, None, "text_encoder", 1)
    return torch.load(path)["base"]


def test_saved_base_loads_strictly_into_transformers(tmp_path):
    transformers = pytest.importorskip("transformers")
    te = tiny_te()
    make_hcpdiff(te, [{"lr": 1e-6, "layers": [""]}], None)
    with torch.no_grad():
        te.text_model.embeddings.token_embedding.weight[5] += 1.0      # "trained"
    base = _saved_base(te, tmp_path)
    assert set(base) == set(R.param_shapes(R.TINY_TE))
    spec = R.TINY_TE
    cfg = transformers.CLIPTextConfig(vocab_size=spec.vocab_size, hidden_size=spec.hidden_size, intermediate_size=spec.intermediate_size,
                                      num_hidden_layers=spec.num_hidden_layers, num_attention_heads=spec.num_attention_heads,
                                      max_position_embeddings=spec.max_position_embeddings, hidden_act="quick_gelu")
    hf = transformers.CLIPTextModel(cfg)
    missing, unexpected = hf.load_state_dict(base, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing)   # a buffer some releases keep in the state dict
    hf.load_state_dict({**hf.state_dict(), **base}, strict=True)
    assert torch.equal(hf.text_model.embeddings.token_embedding.weight, te.text_model.embeddings.token_embedding.weight)


def test_saved_base_of_a_partial_list_is_exactly_the_trainable_parameters(tmp_path):
    te = tiny_te()
    make_hcpdiff(te, [{"layers": ["text_model.encoder.layers.0.mlp", "re:.*final_layer_norm$"]}], None)
    base = _saved_base(te, tmp_path)
    assert set(base) == {n for n, p in te.named_parameters() if p.requires_grad}
    assert set(base) == {f"text_model.encoder.layers.0.mlp.{a}.{b}" for a in ("fc1", "fc2") for b in ("weight", "bias")} | \
        {"text_model.final_layer_norm.weight", "text_model.final_layer_norm.bias"}


def test_optimizer_layouts_take_the_clip_l_token_table():
    """Adafactor factors the [49408, 768] table as any 2-D tensor; AdamW8bit quantizes it in 256-element blocks."""
    shapes = [(49408, 768), (77, 768), (768,)]
    offsets, n = [], 0
    for s in shapes:
        offsets.append(n)
        k = 1
        for d in s:
            k *= d
        n += (k + 3) // 4 * 4
    lay = adafactor.Layout(shapes, offsets, [0, 0, 0])
    assert lay.state_numel == 49408 + 768 + 77 + 768 + 768
    a8 = adamw8bit.Layout([49408 * 768, 77 * 768, 768], offsets, [0, 0, 0], 4096)
    assert a8.nblocks == (49408 * 768 + 255) // 256 + (77 * 768 + 255) // 256 and a8.small_numel == 768
