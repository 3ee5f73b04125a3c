"""Adafactor without a GPU: the fp64 restatement against the real transformers class (stored vectors, and live when transformers
imports), the state layout on the SDXL-base and SD1.5 shapes, the tile walk of the kernels (every element exactly once, never the
padding), the entrypoint's option parsing and the SDXL full fine-tuning config."""
import math
import os

import numpy as np
import pytest
import torch

from hcp_diffusion_b200 import adafactor as A
from hcp_diffusion_b200 import train_ac
from hcp_diffusion_b200.models import UNet2DConditionModel
from hcp_diffusion_b200.utils.config import load_config_with_cli

import adafactor_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SDXL_KW = dict(sample_size=128, block_out_channels=(320, 640, 1280), attention_head_dim=(5, 10, 20), cross_attention_dim=2048,
               down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
               up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"), transformer_layers_per_block=(1, 2, 10),
               use_linear_projection=True, addition_embed_type="text_time", addition_time_embed_dim=256,
               projection_class_embeddings_input_dim=2816)


def run_oracle(case):
    p0, grads = R.golden_inputs(case)
    params = [p.clone() for p in p0]
    states = [{} for _ in params]
    for step_grads in grads:
        for p, g, st in zip(params, step_grads, states):
            R.adafactor_step(p, g, st, **case["opts"])
    return params, states


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


@pytest.mark.parametrize("case", R.GOLDEN_CASES, ids=[c["name"] for c in R.GOLDEN_CASES])
def test_oracle_matches_stored_transformers_vectors(case, golden_dir):
    gold = torch.load(os.path.join(golden_dir, "ref_adafactor.pt"))
    ref = next(c for c in gold["cases"] if c["name"] == case["name"])
    params, states = run_oracle(case)
    for i, (p, q, st, sref) in enumerate(zip(params, ref["params"], states, ref["state"])):
        assert rel(p, q) < 1e-6, (case["name"], R.GOLDEN_SHAPES[i])
        assert st["step"] == sref["step"] == R.GOLDEN_STEPS
        for k in ("exp_avg_sq_row", "exp_avg_sq_col", "exp_avg_sq", "exp_avg"):
            assert (k in st) == (k in sref), k
            if k in st:
                assert rel(st[k], sref[k]) < 1e-6, (case["name"], R.GOLDEN_SHAPES[i], k)


def test_golden_cases_exercise_the_clip_and_the_eps2_floor():
    spike = next(c for c in R.GOLDEN_CASES if c.get("spike"))
    p0, grads = R.golden_inputs(spike)
    params, states = [p.clone() for p in p0], [{} for _ in p0]
    clipped = False
    for step_grads in grads:
        for p, g, st in zip(params, step_grads, states):
            R.adafactor_step(p, g, st)
            if p.dim() >= 2:
                row, col = st["exp_avg_sq_row"], st["exp_avg_sq_col"]
                u = (row / row.mean(-1, keepdim=True)).rsqrt().unsqueeze(-1) * col.unsqueeze(-2).rsqrt() * g.double()
                clipped |= float(u.norm() / math.sqrt(u.numel())) > 1.0
    assert clipped
    zero = next(c for c in R.GOLDEN_CASES if c.get("zero_init"))
    p0, _ = R.golden_inputs(zero)
    assert all(float(p.abs().max()) == 0.0 for p in p0)


def test_oracle_matches_live_transformers():
    tr = pytest.importorskip("transformers.optimization")
    for case in R.GOLDEN_CASES:
        p0, grads = R.golden_inputs(case)
        live = [torch.nn.Parameter(p.clone()) for p in p0]
        opt = tr.Adafactor(live, **case["opts"])
        for step_grads in grads:
            for p, g in zip(live, step_grads):
                p.grad = g.clone()
            opt.step()
        params, _ = run_oracle(case)
        for p, q in zip(params, live):
            assert rel(p, q.detach()) < 1e-6, case["name"]


def test_state_layout_counts_sdxl_and_sd15():
    with torch.device("meta"):
        xl = UNet2DConditionModel(**SDXL_KW)
        sd15 = UNet2DConditionModel()
    shapes = [tuple(p.shape) for p in xl.parameters()]
    assert len(shapes) == 1680 and sum(math.prod(s) for s in shapes) == 2_567_463_684
    assert A.state_numel(shapes) == 244_330_500

    def reference_count(shapes):     # what transformers allocates: exp_avg_sq_row + _col for >= 2 dims, exp_avg_sq otherwise
        return sum((math.prod(s[:-1]) + math.prod(s[:-2] + s[-1:])) if len(s) >= 2 else math.prod(s) for s in shapes)
    s15 = [tuple(p.shape) for p in sd15.parameters()]
    assert A.state_numel(s15) == reference_count(s15) == 457_589_700
    assert A.state_numel([(1280, 640, 1, 1)]) == 2 * 1280 * 640            # a 1x1 conv: row and column states as large as the weight


def walk(layout):
    """numpy restatement of the kernels' element walk (csrc/optim.cu af_for_each): flat indices each item touches."""
    out = []
    for it in layout.items:
        t = layout.tensors[it["tensor"]]
        cw = int(it["c1"] - it["c0"])
        k = A.TILE // cw
        tid = np.arange(A.TILE)
        pi, c = tid // cw, it["c0"] + tid % cw
        for pb in range(int(it["p0"]), int(it["p1"]), k):
            live = pi < min(k, int(it["p1"]) - pb)
            p = pb + pi[live]
            r = np.arange(int(it["r0"]), int(it["r1"]))
            e = ((p[:, None] * int(t["R"]) + r[None, :]) * int(t["C"]) + c[live][:, None]).ravel()
            if not t["factored"]:
                e = e[e < int(t["numel"])]
            out.append(int(t["offset"]) + e)
    return np.concatenate(out)


@pytest.mark.parametrize("extra", [[], [(1280, 5120), (320, 4, 3, 3), (1280, 640, 1, 1), (300, 129), (3, 700, 300)]])
def test_tile_walk_covers_every_element_once_and_no_padding(extra):
    shapes = R.GOLDEN_SHAPES + extra
    offs, n = [], 0
    for s in shapes:
        offs.append(n)
        n += (math.prod(s) + 3) // 4 * 4
    lay = A.Layout(shapes, offs, [0] * len(shapes))
    idx = walk(lay)
    expected = np.concatenate([o + np.arange(math.prod(s)) for s, o in zip(shapes, offs)])
    assert idx.size == expected.size and np.array_equal(np.sort(idx), expected)
    t = lay.tensors
    assert int(t["nitems"].sum()) == lay.items.size and lay.state_numel == A.state_numel(shapes)
    for i, s in enumerate(shapes):                         # row / column scratch only where a tile holds part of a row / column
        f = A.factored_view(s)
        if f:
            assert (t[i]["rowpart"] >= 0) == (f[2] > A.TILE) and (t[i]["colpart"] >= 0) == (f[1] > A.TILE)


def test_options_parsing():
    assert train_ac.optimizer_from_cfg({}) == ("adamw", None)
    assert train_ac.optimizer_from_cfg({"_target_": "torch.optim.AdamW", "lr": 1e-4}) == ("adamw", None)
    name, kw = train_ac.optimizer_from_cfg({"_target_": "transformers.optimization.Adafactor", "_partial_": True,
                                            "relative_step": False, "weight_decay": 1e-3})
    assert name == "adafactor"
    assert kw == {**A.DEFAULTS, "relative_step": False, "weight_decay": 1e-3}
    with pytest.raises(ValueError, match="relative_step"):
        train_ac.optimizer_from_cfg({"_target_": "transformers.optimization.Adafactor", "lr": 1e-3})
    with pytest.raises(ValueError, match="warmup_init"):
        train_ac.optimizer_from_cfg({"_target_": "transformers.optimization.Adafactor", "relative_step": False, "lr": 1e-3,
                                     "warmup_init": True})
    with pytest.raises(TypeError):
        A.check_options({"betas": (0.9, 0.99)})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "torch.optim.SGD"})
    row = A.hyper_row(A.check_options({"beta1": 0.9}), 1e-4, 0.0)
    assert row[5] == pytest.approx(0.9) and int(row[7]) == A.FLAG_SCALE_PARAMETER | A.FLAG_RELATIVE_STEP | A.FLAG_BETA1


def test_schedulers_on_adafactor_push_only_the_lr():
    class Fake:
        optimizer, betas = "adafactor", (0.9, 0.999)
        segments = [{"base_lr": 1e-3}, {"base_lr": 2e-3}]
        pushed = []

        def set_hyper(self, group, lr=None, beta1=None):
            self.pushed.append((group, lr, beta1))
    fake = Fake()
    step = train_ac.make_scheduler({"name": "constant_with_warmup", "num_warmup_steps": 4}, fake)
    step()
    assert fake.pushed[-2:] == [(0, pytest.approx(1e-3 * 0.25), None), (1, pytest.approx(2e-3 * 0.25), None)]
    with pytest.raises(ValueError, match="momentum"):          # as torch refuses cycle_momentum on an optimizer without betas
        train_ac.make_scheduler({"name": "one_cycle", "num_training_steps": 10}, fake)
    train_ac.make_scheduler({"name": "one_cycle", "num_training_steps": 10, "scheduler_kwargs": {"cycle_momentum": False}}, fake)


def test_ft_sdxl_yaml_loads():
    cfg = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "ft_sdxl_synthetic.yaml"))
    assert train_ac.optimizer_from_cfg(cfg.train.optimizer)[0] == "adafactor"
    assert list(cfg.unet[0].layers) == [""]
    kw = {k: v for k, v in cfg.model.unet.items() if k != "_target_"}
    with torch.device("meta"):
        unet = UNet2DConditionModel(**kw)
    assert A.state_numel([tuple(p.shape) for p in unet.parameters()]) == 244_330_500
