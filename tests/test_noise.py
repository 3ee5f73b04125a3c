"""CPU tests of `model.noise_scheduler` (hcp_diffusion_b200/noise.py) and of the float64 restatement of the pyramid noise kernels
(tests/noise_ref.py) against tests/golden/ref_noise.pt, which the unmodified reference PyramidNoiseScheduler and
ZeroTerminalScheduler produced from the same draws (tests/golden/make_golden_noise.py)."""
import json
import os

import numpy as np
import pytest
import torch

import noise_ref as N
from hcp_diffusion_b200 import noise
from hcp_diffusion_b200.engine import ddpm_alphas_cumprod
from hcp_diffusion_b200.train_ac import loss_from_cfg
from hcp_diffusion_b200.utils.config import load_config_with_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DDPM = {"_target_": "diffusers.DDPMScheduler", "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear"}


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "ref_noise.pt"))


def test_restated_pyramid_matches_reference(golden):
    for c in golden["pyramid"]:
        sizes = N.plan(c["seed"], c["draw"], c["group"], c["level"], c["step_size"], c["H"], c["W"])
        assert sizes == [tuple(s) for s in c["sizes"]], (c["sizes"], sizes)
        target, inv_std = N.pyramid(N.golden_base_noise(c).numpy(), sizes, c["discount"], c["seed"], c["draw"], c["group"])
        target = target.reshape(-1)[c["index"].numpy()]
        want = c["target"].double().numpy()
        assert np.abs(target - want).max() <= 1e-6 * np.abs(want).max(), c["sizes"]
        assert abs(inv_std * c["std"] - 1.0) <= 1e-6
        norm = c["normalised"].double().numpy()
        assert np.abs(target * inv_std - norm).max() <= 1e-6 * np.abs(norm).max()
        # the kept quirk: the loss target is the un-normalised sum (std != 1), x_t's noise the normalised one (target / std)
        assert np.abs(want / c["std"] - norm).max() <= 1e-6 * np.abs(norm).max()
        if sizes:
            assert abs(c["std"] - 1.0) > 1e-2


def test_golden_covers_the_issue_cases(golden):
    cases = golden["pyramid"]
    assert {(c["H"], c["W"]) for c in cases} == {(64, 64), (128, 96), (8, 8)}
    assert {c["level"] for c in cases} == {1, 2, 10} and {c["discount"] for c in cases} == {0.5, 0.9}
    assert {c["step_size"] for c in cases} == {1.0, 2.0, 3.0} and {c["B"] for c in cases} == {1, 3}
    assert any(c["sizes"] and c["sizes"][-1][0] == 1 and c["H"] == 8 for c in cases)         # early break on the 8x8 latent


@pytest.mark.parametrize("schedule", ["linear", "scaled_linear", "squaredcos_cap_v2"])
def test_zero_terminal_tables_match_reference(golden, schedule):
    g = golden["zero_terminal"][schedule]
    betas = noise.ddpm_betas(1000, g["beta_start"], g["beta_end"], schedule)
    assert torch.equal(betas, g["betas_in"])
    b64 = N.ddpm_betas(1000, g["beta_start"], g["beta_end"], schedule)
    assert np.all(np.abs(betas.double().numpy() - b64) <= 1e-6 * b64)
    zt = noise.rescale_zero_terminal_snr(betas)
    assert torch.equal(zt, g["betas"])
    sched = noise.resolve({"_target_": "hcpdiff.noise.ZeroTerminalScheduler",
                           "base_scheduler": {"_target_": "diffusers.DDPMScheduler", "beta_start": g["beta_start"], "beta_end": g["beta_end"],
                                              "beta_schedule": schedule}})
    assert torch.equal(sched.alphas_cumprod, g["alphas_cumprod"]) and float(sched.alphas_cumprod[-1]) == 0.0 and sched.zero_terminal
    acp64 = np.cumprod(1.0 - N.zero_terminal(g["betas_in"].double().numpy()))
    assert np.abs(acp64 - g["alphas_cumprod"].double().numpy()).max() < 1e-6


def test_null_key_is_sd1_table_bit_for_bit():
    for cfg in (None,):
        s = noise.resolve(cfg)
        assert torch.equal(s.alphas_cumprod, ddpm_alphas_cumprod()) and s.pyramid is None and s.num_train_timesteps == 1000
    assert torch.equal(noise.resolve(DDPM).alphas_cumprod, ddpm_alphas_cumprod())


def test_every_accepted_form_resolves(tmp_path):
    plain = noise.resolve({"_target_": "diffusers.DDPMScheduler"})
    assert torch.equal(plain.alphas_cumprod, torch.cumprod(1 - torch.linspace(1e-4, 0.02, 1000), 0))
    short = noise.resolve({**DDPM, "num_train_timesteps": 500, "prediction_type": "v_prediction", "clip_sample": False})
    assert short.num_train_timesteps == 500 and torch.equal(short.alphas_cumprod, ddpm_alphas_cumprod(500))
    d = tmp_path / "sd" / "scheduler"
    d.mkdir(parents=True)
    (d / "scheduler_config.json").write_text(json.dumps({"_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012,
                                                         "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000,
                                                         "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1,
                                                         "trained_betas": None, "clip_sample": False}))
    fp = {"_target_": "diffusers.DDPMScheduler.from_pretrained", "pretrained_model_name_or_path": str(tmp_path / "sd"), "subfolder": "scheduler"}
    assert torch.equal(noise.resolve(fp).alphas_cumprod, ddpm_alphas_cumprod())
    zt = {"_target_": "hcpdiff.noise.ZeroTerminalScheduler", "base_scheduler": DDPM}
    pz = noise.resolve({"_target_": "hcpdiff.noise.PyramidNoiseScheduler", "base_scheduler": zt})
    assert pz.pyramid == {"level": 10, "discount": 0.9, "step_size": 2.0} and pz.zero_terminal
    assert torch.equal(pz.alphas_cumprod, noise.resolve(zt).alphas_cumprod)
    pf = noise.resolve({"_target_": "hcpdiff.noise.PyramidNoiseScheduler", "level": 6, "discount": 0.8, "step_size": 1.5,
                        "base_scheduler": {**fp, "_partial_": False}})
    assert pf.pyramid == {"level": 6, "discount": 0.8, "step_size": 1.5} and not pf.zero_terminal
    rz = noise.resolve({**DDPM, "rescale_betas_zero_snr": True})
    assert torch.equal(rz.alphas_cumprod, noise.resolve(zt).alphas_cumprod)


def test_refusals_name_their_cause(tmp_path):
    zt = {"_target_": "hcpdiff.noise.ZeroTerminalScheduler", "base_scheduler": DDPM}
    pyr = {"_target_": "hcpdiff.noise.PyramidNoiseScheduler", "base_scheduler": DDPM}
    cases = [
        ({"_target_": "diffusers.EulerDiscreteScheduler"}, NotImplementedError, "EulerDiscreteScheduler"),
        ({**DDPM, "trained_betas": [0.1] * 1000}, NotImplementedError, "trained_betas"),
        ({**DDPM, "beta_schedule": "sigmoid"}, NotImplementedError, "sigmoid"),
        ({**DDPM, "betas": 1}, TypeError, "betas"),
        ({"_target_": "diffusers.DDPMScheduler.from_pretrained", "pretrained_model_name_or_path": str(tmp_path), "subfolder": "scheduler"},
         FileNotFoundError, "scheduler_config.json"),
        ({**pyr, "resize_mode": "nearest"}, NotImplementedError, "resize_mode"),
        ({**pyr, "level": 0}, ValueError, "level"),
        ({**pyr, "level": 17}, ValueError, "level"),
        ({**pyr, "step_size": 0.5}, ValueError, "step_size"),
        ({**pyr, "base_scheduler": pyr}, NotImplementedError, "PyramidNoiseScheduler around"),
        ({"_target_": "hcpdiff.noise.ZeroTerminalScheduler", "base_scheduler": pyr}, NotImplementedError, "ZeroTerminalScheduler around"),
    ]
    for cfg, exc, msg in cases:
        with pytest.raises(exc, match=msg):
            noise.resolve(cfg)
    for loss in ({"type": "EDMLoss", "gamma": 1.0}, "edm"):
        with pytest.raises(ValueError, match="EDMLoss"):
            noise.resolve(zt, loss)
        with pytest.raises(ValueError, match="EDMLoss"):
            noise.resolve({**DDPM, "rescale_betas_zero_snr": True}, loss)
    noise.resolve(DDPM, {"type": "EDMLoss"})                      # EDM on a table without a zero is fine
    for kind in ("MinSNRLoss", "SoftMinSNRLoss", "KDiffMinSNRLoss"):
        noise.resolve(zt, {"type": kind, "gamma": 5.0})


def test_pyramid_ztsnr_yaml():
    conf = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "lora_pyramid_ztsnr_sd15_synthetic.yaml"), args_list=[])
    loss = loss_from_cfg(conf.train.get("loss"))
    assert loss == {"type": "MinSNRLoss", "gamma": 5.0}
    s = noise.resolve(conf.model.noise_scheduler, loss)
    assert s.pyramid == {"level": 10, "discount": 0.9, "step_size": 2.0} and s.zero_terminal and s.num_train_timesteps == 1000
    assert conf.lora_unet[0]["rank"] == 8
