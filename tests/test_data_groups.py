"""CPU tests of the `data` section with data groups: the flat form parses as before, the reference's dict of datasets gives groups,
loss weights and the summed `scale_lr` factor, and cfgs/train/dreambooth_sd15_synthetic.yaml mirrors the reference's DreamBooth.yaml."""
import os

import pytest

from hcp_diffusion_b200.train_ac import data_groups, images_per_step
from hcp_diffusion_b200.utils.config import load_config_with_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", ["lora_sd15_synthetic", "lora_te_sd15_synthetic", "lora_sdxl_te_synthetic", "ft_sdxl_synthetic"])
def test_flat_data_form_is_unchanged(name):
    conf = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", f"{name}.yaml"), args_list=[])
    assert data_groups(conf.data) is None
    assert images_per_step(conf.data) == int(conf.data["batch_size"])


def test_flat_form_without_batch_size_defaults_to_four():
    assert data_groups({}) is None and images_per_step({}) == 4
    assert data_groups({"path": "x.pt", "num_samples": 8}) is None and images_per_step({"path": "x.pt"}) == 4
    # a top-level batch_size keeps the flat form whatever else is there
    assert data_groups({"batch_size": 2, "extra": {"batch_size": 1}}) is None


def test_nested_form_gives_groups_weights_and_summed_batch():
    data = {"dataset1": {"batch_size": 4, "path": "a.pt"}, "dataset_class": {"batch_size": 1, "loss_weight": 0.25, "num_samples": 8}}
    groups = data_groups(data)
    assert [(n, bs, w) for n, _, bs, w in groups] == [("dataset1", 4, 1.0), ("dataset_class", 1, 0.25)]
    assert groups[0][1]["path"] == "a.pt" and groups[1][1]["num_samples"] == 8
    assert images_per_step(data) == 5
    with pytest.raises(ValueError):
        data_groups({"dataset1": {"batch_size": 0}})


def test_dreambooth_yaml_mirrors_reference_items():
    conf = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "dreambooth_sd15_synthetic.yaml"), args_list=[])
    assert len(conf.unet) == 1 and float(conf.unet[0]["lr"]) == 1e-6 and conf.unet[0]["layers"] == [""] and not conf.get("lora_unet")
    assert conf.train.gradient_accumulation_steps == 1 and conf.train.save_step == 100
    sch = conf.train.scheduler
    assert (sch.name, sch.num_warmup_steps, sch.num_training_steps) == ("constant_with_warmup", 50, 600)
    groups = data_groups(conf.data)
    assert [(n, bs, w) for n, _, bs, w in groups] == [("dataset1", 4, 1.0), ("dataset_class", 1, 1.0)]
    assert images_per_step(conf.data) == 5


def test_data_group_overrides_from_the_command_line():
    conf = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "dreambooth_sd15_synthetic.yaml"),
                                args_list=["data.dataset_class.loss_weight=0.5", "data.dataset1.batch_size=2"])
    groups = data_groups(conf.data)
    assert [(bs, w) for _, _, bs, w in groups] == [(2, 1.0), (1, 0.5)] and images_per_step(conf.data) == 3
