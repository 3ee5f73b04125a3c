"""AdamW8bit without a GPU: the restatement in tests/adamw8bit_ref.py against a hand-computed two-step case, the structure of the two
code maps, the layout of hcp_diffusion_b200.adamw8bit (the 8-bit threshold, partial blocks, blocks counted per tensor), the engine's
state and defaults, the entrypoint's option parsing and refusals, and the SDXL AdamW8bit fine-tuning config."""
import math
import os

import numpy as np
import pytest
import torch

from hcp_diffusion_b200 import adamw8bit as A
from hcp_diffusion_b200 import train_ac
from hcp_diffusion_b200.engine import LoraTrainStep
from hcp_diffusion_b200.utils.config import load_config_with_cli

import adamw8bit_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A8 = "bitsandbytes.optim.AdamW8bit"


def top_signed(k):        # entry k of the signed map's top decade: midpoints of linspace(0.1, 1, 65)
    return 0.1 + 0.9 * (k + 0.5) / 64


def unsigned_decade(i, k):  # entry k of the unsigned map's decade 10^(i-6): midpoints of linspace(0.1, 1, 2^(i+1) + 1)
    return 10.0 ** (i - 6) * (0.1 + 0.9 * (k + 0.5) / 2 ** (i + 1))


def test_restatement_known_answer_two_steps():
    """lr 0.5, betas (0.5, 0.75), eps 0, min_8bit_size 4: W (4 elements, one partial block) is 8-bit, wd 0; b (2 elements) keeps fp32
    moments, wd 0.5 (p x 0.75 after each step).  Step 1 starts from zero state (absmax 0), so every value is dyadic; its codes are
    the map entries nearest to s / absmax.  Step 2 decodes those entries (values of the form 0.1 + 0.9 (k + 0.5) / 2^j) and has a
    zero gradient, a sign change of s1 and a NaN gradient (moments to 0, p unchanged)."""
    W = torch.nn.Parameter(torch.ones(4))
    b = torch.nn.Parameter(torch.full((2,), 2.0))
    opt = R.AdamW8bit([{"params": [W], "weight_decay": 0.0}, {"params": [b], "weight_decay": 0.5}], lr=0.5, betas=(0.5, 0.75), eps=0.0,
                      min_8bit_size=4)
    # step 1: s1 = g / 2, s2 = g^2 / 4, corr1 = corr2 = 1/2, step size -1/2: p = 1 - sign(g) / 2
    W.grad, b.grad = torch.tensor([1.0, -1.0, 2.0, 4.0]), torch.tensor([4.0, -2.0])
    opt.step()
    sw, sb = opt.state[W], opt.state[b]
    assert W.tolist() == [0.5, 1.5, 0.5, 0.5]
    assert b.tolist() == [0.75 * 1.5, 0.75 * 2.5]                           # the decay comes after the step
    assert sb["state1"].tolist() == [2.0, -1.0] and sb["state2"].tolist() == [4.0, 1.0]
    assert sw["absmax1"].tolist() == [2.0] and sw["absmax2"].tolist() == [4.0]
    # s1 / 2 = (0.25, -0.25, 0.5, 1): top-decade k = 10, 10 (negative: index 63 - k), 28, and 1.0 at 255
    # s2 / 4 = (1/16, 1/16, 1/4, 1): unsigned decade 10^-1 k = 37 (index 63 + k), decade 10^0 k = 21 (index 127 + k), 1.0 at 255
    assert sw["state1"].tolist() == [191 + 10, 63 - 10, 191 + 28, 255]
    assert sw["state2"].tolist() == [63 + 37, 63 + 37, 127 + 21, 255]
    # step 2: g = (0, 0, -2, nan) for W, (0, 2) for b
    W.grad, b.grad = torch.tensor([0.0, 0.0, -2.0, float("nan")]), torch.tensor([0.0, 2.0])
    opt.step()
    d1 = [2 * top_signed(10), -2 * top_signed(10), 2 * top_signed(28)]
    d2 = [4 * unsigned_decade(5, 37), 4 * unsigned_decade(5, 37), 4 * unsigned_decade(6, 21)]
    s1 = [0.5 * d1[0], 0.5 * d1[1], 0.5 * d1[2] - 1.0, 0.0]
    s2 = [0.75 * d2[0], 0.75 * d2[1], 0.75 * d2[2] + 1.0, 0.0]
    step_size = -0.5 * math.sqrt(1 - 0.75 ** 2) / (1 - 0.5 ** 2)
    want_w = [p + step_size * m / math.sqrt(v) for p, m, v in zip([0.5, 1.5, 0.5], s1, s2)] + [0.5]
    assert W.tolist() == pytest.approx(want_w, rel=1e-6)
    assert sw["absmax1"].tolist() == pytest.approx([abs(s1[2])], rel=1e-6) and sw["absmax2"].tolist() == pytest.approx([s2[2]], rel=1e-6)
    # s1 / absmax1 = (0.496, -0.496, -1, 0): k = 28, 63 - 28, the most negative entry (index 0), and 0 at index 127
    # s2 / absmax2 = (0.1073, 0.1073, 1, 0): above the midpoint of the top decade's first two entries, so k = 1 (index 128)
    assert sw["state1"].tolist() == [191 + 28, 63 - 28, 0, 127]
    assert sw["state2"].tolist() == [128, 128, 255, 0]
    m_b, v_b = [1.0, 0.5], [3.0, 1.75]
    want_b = [0.75 * (p + step_size * m / math.sqrt(v)) for p, m, v in zip([1.125, 1.875], m_b, v_b)]
    assert sb["state1"].tolist() == m_b and sb["state2"].tolist() == v_b
    assert b.tolist() == pytest.approx(want_b, rel=1e-6)


def test_restatement_sign_fix_and_all_zero_block():
    """A first moment of -0.0 (a zero gradient on fresh state is +0; an explicit -0.0 gradient keeps the sign bit) maps to the 0
    entry, whose sign bit differs, so its code moves one step down to the smallest negative entry; an all-zero block keeps scale 0
    and encodes 0."""
    n = 300                                                          # two blocks, the second partial (44 elements)
    p = np.ones(n, np.float32)
    g = np.zeros(n, np.float32)
    g[:256] = np.linspace(-1, 1, 256, dtype=np.float32)
    g[5] = -0.0
    c = np.zeros(n, np.uint8)
    am = np.zeros(2, np.float32)
    pn, k1, k2, n1, n2, s1, _ = R.step_8bit(p, g, c, c, am, am, (1e-3, 0.9, 0.999, 1e-8, 0.0), 1)
    assert np.signbit(s1[5]) and s1[5] == 0
    zero_code = int(np.flatnonzero(R.MAP1 == 0)[0])
    assert k1[5] == zero_code - 1 and R.MAP1[k1[5]] < 0
    assert n1[1] == 0 and n2[1] == 0 and (k1[256:] == zero_code).all() and (k2[256:] == 0).all()
    assert (pn[256:] == 1).all()


def test_dynamic_maps_structure():
    m1, m2 = A.create_dynamic_map(True), A.create_dynamic_map(False)
    assert m1.dtype == m2.dtype == torch.float32 and m1.numel() == m2.numel() == 256
    assert bool((m1.diff() > 0).all()) and bool((m2.diff() > 0).all())       # sorted, no repeats
    assert float(m1[255]) == 1.0 and float(m2[255]) == 1.0 and float(m2[0]) == 0.0
    assert int((m1 < 0).sum()) == 127 and int((m1 == 0).sum()) == 1 and float(m1[127]) == 0.0
    assert float(m1[0]) == pytest.approx(-top_signed(63), rel=1e-6)          # no -1: the most negative code is -0.99297
    # the signed map mirrors its positive side (without 1.0); per decade 10^(i-6): 2^i signed entries, 2^(i+1) unsigned
    assert torch.equal(-m1[:127].flip(0), m1[128:255])
    for i in range(7):
        lo, hi = 10.0 ** (i - 6) * 0.1, 10.0 ** (i - 6)
        assert int(((m1 > lo) & (m1 < hi)).sum()) == 2 ** i
        assert int(((m2 > lo) & (m2 < hi)).sum()) == 2 ** (i + 1)
    assert float(m2[127 + 21]) == pytest.approx(unsigned_decade(6, 21), rel=1e-6)
    assert torch.equal(A.maps(), torch.stack([m1, m2]))


def test_quantize_is_nearest_with_last_probe_ties():
    rng = np.random.default_rng(0)
    for code, signed in ((R.MAP1, True), (R.MAP2, False)):
        x = rng.uniform(-1 if signed else 0, 1, 20000).astype(np.float32)
        x = np.concatenate([x, code, [np.float32(-1) if signed else np.float32(0), np.float32(1)]]).astype(np.float32)
        k = R.quantize(code, x, signed)
        dist = np.abs(code[k].astype(np.float64) - x)
        best = np.abs(code[None, :].astype(np.float64) - x[:, None]).min(axis=1)
        assert np.all(dist <= best + 1e-7)
        assert np.array_equal(R.quantize(code, code, signed), np.arange(256))     # every entry encodes to itself
    # an exact fp32 midpoint goes to the last probed entry: at the top of the map that is the lower one of the pair
    mid = np.float32((R.MAP2[254] + R.MAP2[255]) * np.float32(0.5))
    assert R.quantize(R.MAP2, np.array([mid]), False)[0] == 254


def test_layout_threshold_partial_blocks_and_per_tensor_blocks():
    numels = [4095, 4096, 4097, 7, 300, 256 * 64 * 2 + 1]
    offsets, off = [], 4                                   # flat offsets are multiples of 4, not of 256
    for n in numels:
        offsets.append(off)
        off += (n + 3) // 4 * 4
    lay = A.Layout(numels, offsets, [0, 0, 1, 1, 0, 1], min_8bit_size=4096)
    t = lay.tensors
    assert t["mode"].tolist() == [0, 1, 1, 0, 0, 1]
    assert t["offset"].tolist() == offsets and t["numel"].tolist() == numels and t["group"].tolist() == [0, 0, 1, 1, 0, 1]
    # 8-bit: codes from multiples of 16, one absmax per 256 elements counted from the tensor's own first element
    assert t["state"][t["mode"] == 1].tolist() == [0, 4096, 4096 + 4112] and lay.code_bytes == 4096 + 4112 + 32784
    assert t["absmax"][t["mode"] == 1].tolist() == [0, 16, 16 + 17] and lay.nblocks == 16 + 17 + 129
    # 32-bit: m / v from multiples of 4
    assert t["state"][t["mode"] == 0].tolist() == [0, 4096, 4104] and lay.small_numel == 4096 + 8 + 300
    assert (t["absmax"][t["mode"] == 0] == -1).all()
    # items: whole blocks of one tensor, at most 64, tiling every tensor once in order
    it = lay.items
    for i, n in enumerate(numels):
        mine = it[it["tensor"] == i]
        nb = -(-n // 256)
        assert mine["block0"].tolist() == list(range(0, nb, 64)) and mine["block1"][-1] == nb
        assert ((mine["block1"] - mine["block0"]) <= 64).all()
    assert it["tensor"].tolist() == sorted(it["tensor"].tolist())
    assert lay.state_bytes == 2 * lay.code_bytes + 8 * lay.nblocks + 8 * lay.small_numel
    assert lay.bytes_per_step() == 16 * (4096 + 4097 + 32769) + 16 * lay.nblocks + 28 * (4095 + 7 + 300)
    assert A.Layout([4096], [0], [0], min_8bit_size=4097).tensors["mode"].tolist() == [0]
    assert A.Layout([1], [0], [0], min_8bit_size=0).tensors["mode"].tolist() == [1]
    with pytest.raises(ValueError):
        A.Layout([0], [0], [0])


def test_options_parsing_defaults_and_refusals():
    assert train_ac.optimizer_from_cfg({"_target_": A8, "_partial_": True}) == \
        ("adamw8bit", {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 1e-2, "min_8bit_size": 4096})
    name, opts = train_ac.optimizer_from_cfg({"_target_": A8, "lr": 3e-5, "betas": [0.95, 0.98], "eps": 1e-6, "weight_decay": 1e-3,
                                              "min_8bit_size": 16384, "amsgrad": False, "optim_bits": 8, "args": None,
                                              "percentile_clipping": 100, "block_wise": True, "is_paged": False})
    assert name == "adamw8bit"
    assert opts == {"lr": 3e-5, "betas": (0.95, 0.98), "eps": 1e-6, "weight_decay": 1e-3, "min_8bit_size": 16384}
    with pytest.raises(TypeError, match="foo"):
        train_ac.optimizer_from_cfg({"_target_": A8, "foo": 1})
    for key, value in (("percentile_clipping", 95), ("block_wise", False), ("amsgrad", True), ("is_paged", True),
                       ("args", {"optim_bits": 8})):
        with pytest.raises(NotImplementedError, match=key):
            train_ac.optimizer_from_cfg({"_target_": A8, key: value})
    for other in ("bitsandbytes.optim.Adam8bit", "bitsandbytes.optim.Lion8bit", "bitsandbytes.optim.PagedAdamW8bit",
                  "bitsandbytes.optim.AdamW"):
        with pytest.raises(NotImplementedError, match="bitsandbytes.optim.AdamW8bit"):
            train_ac.optimizer_from_cfg({"_target_": other})
    with pytest.raises(NotImplementedError):
        train_ac.optimizer_from_cfg({"_target_": "somewhere.else.AdamW8bit"})
    with pytest.raises(ValueError, match="betas"):
        A.check_options({"betas": (0.9,)})


def cpu_step(optimizer, **kw):
    params = [torch.nn.Parameter(torch.zeros(5)), torch.nn.Parameter(torch.zeros(64, 80)), torch.nn.Parameter(torch.zeros(3, 2))]
    return LoraTrainStep(torch.nn.Identity(), [{"params": params[:2], "lr": 1e-4}, {"params": [params[2]], "lr": 2e-4}],
                         optimizer=optimizer, **kw)


def test_engine_adamw8bit_state_and_defaults():
    a8 = cpu_step("adamw8bit")
    lay = a8.a8_layout
    assert a8.m is None and a8.v is None
    assert lay.tensors["mode"].tolist() == [0, 1, 0] and lay.code_bytes == 5120 and lay.nblocks == 20 and lay.small_numel == 8 + 8
    assert a8.optimizer_state_bytes == 2 * 5120 + 2 * 4 * 20 + 2 * 4 * 16
    assert [b.data_ptr() for b in a8._opt_buffers()] == [b.data_ptr() for b in (a8.a8_codes, a8.a8_absmax, a8.a8_state32, a8.a8_steps)]
    assert a8.betas == (0.9, 0.999)
    for gi, (s, lr) in enumerate(zip(a8.segments, (1e-4, 2e-4))):
        assert s["hyper"].tolist() == pytest.approx([lr, 0.9, 0.999, 1e-8, 1e-2])
        assert s["hyper"].data_ptr() == a8.a8_hyper[gi].data_ptr() and s["step"].data_ptr() == a8.a8_steps[gi:].data_ptr()
    assert a8.step_count.data_ptr() == a8.a8_steps.data_ptr()
    a8.set_hyper(1, lr=5e-5, beta1=0.85)
    assert a8.a8_hyper[1].tolist()[:2] == pytest.approx([5e-5, 0.85])
    assert torch.equal(a8.a8_maps.cpu(), A.maps())
    kw = cpu_step("adamw8bit", optimizer_kwargs={"betas": (0.95, 0.98), "weight_decay": 0.0, "eps": 1e-6, "min_8bit_size": 4})
    assert kw.a8_layout.tensors["mode"].tolist() == [1, 1, 1]
    assert kw.segments[0]["hyper"].tolist() == pytest.approx([1e-4, 0.95, 0.98, 1e-6, 0.0])
    explicit = cpu_step("adamw8bit", betas=(0.8, 0.9), weight_decay=1e-3, lr=1e-3)
    assert explicit.segments[0]["hyper"].tolist() == pytest.approx([1e-4, 0.8, 0.9, 1e-8, 1e-3])
    with pytest.raises(NotImplementedError, match="percentile_clipping"):
        cpu_step("adamw8bit", optimizer_kwargs={"percentile_clipping": 5})
    with pytest.raises(TypeError):
        cpu_step("adamw8bit", optimizer_kwargs={"momentum": 0.9})
    # AdamW and Lion are unchanged: no optimizer_kwargs, their own defaults
    adamw = cpu_step("adamw")
    assert adamw.optimizer_state_bytes == 2 * 4 * adamw.flat.numel
    with pytest.raises(ValueError, match="optimizer_kwargs"):
        cpu_step("adamw", optimizer_kwargs={"weight_decay": 1e-2})
    with pytest.raises(ValueError, match="optimizer_kwargs"):
        cpu_step("lion", optimizer_kwargs={"weight_decay": 1e-2})
    with pytest.raises(ValueError, match="adamw8bit"):
        cpu_step("adam8bit")


def test_ft_adamw8bit_sdxl_yaml_loads():
    cfg = load_config_with_cli(os.path.join(ROOT, "cfgs", "train", "ft_adamw8bit_sdxl_synthetic.yaml"))
    name, opts = train_ac.optimizer_from_cfg(cfg.train.optimizer)
    assert name == "adamw8bit" and opts["weight_decay"] == 1e-3 and opts["betas"] == (0.9, 0.999)
    assert list(cfg.unet[0].layers) == [""] and float(cfg.unet[0].lr) == 1e-6
    assert cfg.model.unet.addition_embed_type == "text_time" and list(cfg.model.unet.block_out_channels) == [320, 640, 1280]
    assert cfg.model.unet.sample_size == 128 and cfg.train.max_grad_norm == 1.0
