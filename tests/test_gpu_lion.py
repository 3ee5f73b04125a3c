"""Lion on the GPU (`pytest -m gpu`): hcp_lion_flat_dev against a float64 restatement at its edges, and the training step with
optimizer='lion' against oracle.step_ref.ReferenceLoop running tests/lion_ref.Lion, and the entrypoint on a tiny copy of
cfgs/train/ft_lion_sd15_synthetic.yaml.

Kernel: four steps from the kernel's own state, each against float64 computed from the exact fp32 values the kernel reads (the
clip factor and the scaled gradient rounded as the kernel rounds them).  m' within LION_M of |beta2 m| + |(1 - beta2) g| (a few
fp32 ulp); p' within one fp32 ulp (of the larger of p (1 - lr wd) and p') of p (1 - lr wd) - lr sign(c); where |c| is within
rounding of 0 every sign is accepted; elements with g = m = 0 are exactly p (1 - lr wd) rounded once.

Training step: Lion moves every parameter by +-lr (plus the decay), so the update (after - before) of each model is compared by its
direction cosine, which is the share of parameters whose sign(c) agrees with the reference (1 - 2 x the share that flips).  Signs flip
where |c| is below the bf16 noise of the gradient, so the bound sits under the worst cosine measured on one H100 80GB HBM3 (700 W).
Kernel errors measured there: m' 1.15e-7, p' 0.5 ulp.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():          # fp32 torch references must be real fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.engine import LoraTrainStep  # noqa: E402
from hcp_diffusion_b200.models import CLIPTextModel, UNet2DConditionModel  # noqa: E402
from hcp_diffusion_b200.utils.cfg_net_tools import make_hcpdiff  # noqa: E402
from oracle import step_ref as S  # noqa: E402
from oracle import unet_ref as U  # noqa: E402

import clip_ref as CR  # noqa: E402
import lion_ref as L  # noqa: E402

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HCP_ERR_INVALID = -1
F32 = np.float32

LION_M = 2.4e-7                 # m': |got - ref| / (|b2 m| + |(1 - b2) g|), 4 fp32 ulp
LION_P_ULP = 1.0                # p': fp32 ulps of max(|p (1 - lr wd)|, |p'|)
COS = 0.96                      # update cosine per model; measured 0.9871 (LoRA), 0.9876 (full fine-tune), 0.9906 / 0.9940 (UNet /
                                # text-encoder adapters of the joint step)


def measured(name: str, value: float, bound: float, above: bool = False) -> None:
    print(f"MEASURED {name}: {value:.6e} ({'>=' if above else '<='} {bound:.2e})")
    assert (value >= bound) if above else (value <= bound), f"{name}: {value:.6e} vs {bound:.2e}"


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def gen(seed: int) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(seed)


class FlatCanary:
    """fp32 [lo + n + 8] prefilled with all-ones bits; `view` = elements [lo, lo + n); `check()`: nothing outside was written."""

    def __init__(self, n: int, lo: int = 8, values=None):
        self.buf = torch.full((lo + n + 8,), -1, dtype=torch.int32, device=DEV).view(torch.float32)
        self.view = self.buf[lo:lo + n]
        if values is not None:
            self.view.copy_(values)
        self.lo, self.n = lo, n

    def check(self, name: str) -> None:
        b = self.buf.view(torch.int32)
        stray = int((b[:self.lo] != -1).sum()) + int((b[self.lo + self.n:] != -1).sum())
        assert stray == 0, f"{name}: {stray} elements outside [lo, lo + n) were written"


# the four steps: (hyper = lr, beta1, beta2, eps (unused), weight_decay), grad_scale, clip (None: max_norm = 0; otherwise
# max_norm = clip x ||g grad_scale||, so < 1 engages it).  lr and beta1 are rewritten between steps, as OneCycleLR does.
LION_STEPS = [((1e-3, 0.9, 0.99, 1e-8, 1e-2), 0.5, 0.3),
              ((5e-4, 0.85, 0.99, 1e-8, 0.0), 1.0, 3.0),
              ((2e-3, 0.95, 0.98, 1e-6, 1e-2), 0.5, None),
              ((1e-3, 0.9, 0.99, 1e-8, 0.0), 1.0, 0.5)]

# (n, lo): n < 0 stands for 4 (cap4 + d) + r with d = -n // 4 - 2 and r = -n % 4, cap4 = 256 x 16 x SMs float4 (one grid-stride
# wave of hcp_lion_flat_dev; the SM count is only known on the device)
LION_SIZES = [(n, 8) for n in (1, 2, 3, 4, 5)] + [(-(4 * (d + 2) + r), 8) for d in (-1, 0, 1) for r in (0, 1, 3)]
LION_SIZES.append((1000003, 36))                              # a segment at flat + 4 lo, lo % 4 == 0 and lo % 256 != 0


def lion_n(n: int) -> int:
    if n > 0:
        return n
    d, r = -n // 4 - 2, -n % 4
    return 4 * (256 * 16 * sms() + d) + r


def kernel_scale(gscale: float, sumsq: float, max_norm: float) -> np.float32:
    """gscale x clip as the kernel computes it in fp32 (af_grad_scale)."""
    gs, mn = F32(gscale), F32(max_norm)
    clip = F32(1.0)
    if mn > 0:
        norm = F32(np.sqrt(F32(sumsq))) * gs
        clip = min(F32(1.0), F32(mn / F32(norm + F32(1e-6))))
    return F32(gs * clip)


def lion_check(p0, g, m0, p1, m1, hyper32, gs):
    """Errors of one kernel step against float64 from the fp32 inputs: (worst m' error, worst p' error in ulps, share of elements
    with an ambiguous sign, bool mask of g = m = 0)."""
    lr, b1, b2, _, wd = (F32(h) for h in hyper32)
    decay = F32(F32(1.0) - F32(lr * wd))
    grad32 = (g * gs).astype(F32)                                # the kernel's g * grad_scale, rounded once
    gd, md, pd0 = grad32.astype(np.float64), m0.astype(np.float64), p0.astype(np.float64)
    omb1, omb2 = float(F32(1.0) - b1), float(F32(1.0) - b2)
    c = float(b1) * md + omb1 * gd
    m_ref = float(b2) * md + omb2 * gd
    m_scale = np.abs(float(b2) * md) + np.abs(omb2 * gd)
    m_abs = np.abs(m1.astype(np.float64) - m_ref)
    m_err = np.divide(m_abs, m_scale, out=np.where(m_abs > 0, np.inf, 0.0), where=m_scale > 0)
    pdec = pd0 * float(decay)
    ulp = np.spacing(np.maximum(np.abs(pdec), np.abs(p1.astype(np.float64))).astype(F32)).astype(np.float64)
    near0 = np.abs(c) <= 2.0 ** -22 * (np.abs(float(b1) * md) + np.abs(omb1 * gd))
    errs = [np.abs(p1.astype(np.float64) - (pdec - float(lr) * s)) / ulp for s in (-1.0, 0.0, 1.0)]
    exact = np.abs(p1.astype(np.float64) - (pdec - float(lr) * np.sign(c))) / ulp
    p_err = np.where(near0, np.minimum(np.minimum(errs[0], errs[1]), errs[2]), exact)
    zero = (g == 0) & (m0 == 0)
    assert np.array_equal(p1[zero].view(np.int32), (p0[zero] * decay).astype(F32).view(np.int32)), "g = m = 0 must only decay p"
    assert not np.any(m1[zero]), "g = m = 0 must leave m = 0"
    return float(m_err.max(initial=0.0)), float(p_err.max(initial=0.0)), float(near0.mean()), zero


def run_lion(n, lo, seed=0, check=True):
    g = gen(seed)
    p = FlatCanary(n, lo, torch.randn(n, generator=g, device=DEV))
    m = FlatCanary(n, lo, 0.1 * torch.randn(n, generator=g, device=DEV))
    zero = torch.rand(n, generator=g, device=DEV) < 1 / 16     # g = m = 0 at every step: c = 0 exactly, p only decays
    m.view[zero] = 0.0
    grad = FlatCanary(n, lo)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    hyper = torch.zeros(5, device=DEV)
    sumsq = torch.zeros(1, device=DEV)
    worst, ambiguous = [0.0, 0.0], 0.0
    for k, (hy, gscale, clip) in enumerate(LION_STEPS, start=1):
        gv = torch.randn(n, generator=g, device=DEV) * (1 + k)
        gv[zero] = 0.0
        grad.view.copy_(gv)
        hyper.copy_(torch.tensor(hy))
        sumsq.fill_(float(grad.view.double().square().sum()))
        ss = float(sumsq)
        max_norm = 0.0 if clip is None else clip * math.sqrt(ss) * gscale
        before = [t.view.cpu().numpy().copy() for t in (p, m)]
        call("hcp_lion_flat_dev", p.view.data_ptr(), grad.view.data_ptr(), m.view.data_ptr(), n, hyper.data_ptr(), gscale,
             sumsq.data_ptr(), max_norm, step.data_ptr(), stream_ptr())
        assert int(step) == k
        if check:
            gs = kernel_scale(gscale, ss, max_norm)
            if clip is not None and clip < 1 and ss > 0:
                assert gs < F32(gscale), "the clip must be engaged"
            em, ep, amb, zmask = lion_check(before[0], grad.view.cpu().numpy(), before[1], p.view.cpu().numpy(), m.view.cpu().numpy(),
                                            [float(h) for h in hyper.cpu()], gs)
            worst = [max(worst[0], em), max(worst[1], ep)]
            ambiguous = max(ambiguous, amb)
            assert n < 64 or zmask.any()
    for t, name in zip((p, m, grad), "pmg"):
        t.check(f"lion n={n} {name}")
    return worst, ambiguous, (p.view.clone(), m.view.clone())


@pytest.mark.parametrize("n,lo", LION_SIZES)
def test_lion_flat_dev_per_step(n, lo):
    """hcp_lion_flat_dev four steps from its own state, each step against the float64 restatement: tail-only sizes (n < 4), one
    grid-stride wave of 256 x 16 x SMs float4 exactly / -1 / +1 with n % 4 in {0, 1, 3}, an offset segment of the flat buffer with
    untouched neighbours, the clip engaged and not, grad_scale 1/2, lr and beta1 rewritten between steps."""
    n = lion_n(n)
    (wm, wp), amb, _ = run_lion(n, lo)
    print(f"lion n={n}: share of elements with |c| within rounding of 0: {amb:.2e}")
    measured(f"lion n={n} lo={lo} m", wm, LION_M)
    measured(f"lion n={n} lo={lo} p ulps", wp, LION_P_ULP)


def test_lion_flat_dev_bit_identical_repeats():
    n = lion_n(-(4 * 3 + 3))
    _, _, a = run_lion(n, 8, seed=5, check=False)
    _, _, b = run_lion(n, 8, seed=5, check=False)
    assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def rc_of(*args):
    rc = _lib.lib().hcp_lion_flat_dev(*args)
    torch.cuda.synchronize()
    return rc


def test_lion_refusals_before_launch_and_empty_size():
    """Null pointers, n < 0 and a buffer off 16-byte alignment are refused before any launch (the step counter stays); n == 0 is a
    no-op that launches nothing."""
    buf = torch.full((3, 64), 1.5, device=DEV)                  # p, g, m rows of 256 bytes
    hyper = torch.tensor([1e-3, 0.9, 0.99, 1e-8, 1e-2], device=DEV)
    step = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    P, G, M = (buf[j].data_ptr() for j in range(3))
    H, T, SS = hyper.data_ptr(), step.data_ptr(), stream_ptr()
    before = _lib.launch_count
    cases = [(P + 4, G, M, 8), (P, G + 8, M, 8), (P, G, M + 12, 8), (P, G, M, -1),
             (None, G, M, 8), (P, None, M, 8), (P, G, None, 8)]
    for p, g, m, n in cases:
        assert rc_of(p, g, m, n, H, 1.0, None, 0.0, T, SS) == HCP_ERR_INVALID, (p, g, m, n)
    assert rc_of(P, G, M, 8, None, 1.0, None, 0.0, T, SS) == HCP_ERR_INVALID
    assert rc_of(P, G, M, 8, H, 1.0, None, 0.0, None, SS) == HCP_ERR_INVALID
    assert rc_of(P, G, M, 0, H, 1.0, None, 0.0, T, SS) == 0
    assert _lib.launch_count == before
    assert int(step) == 3 and bool((buf == 1.5).all())


# ----------------------------------------------------------------------------------------------------------------------------------
# the training step against the reference loop
# ----------------------------------------------------------------------------------------------------------------------------------
LR, WD = 1e-4, 1e-2


def tiny_unet(sd, spec=U.TINY):
    u = UNet2DConditionModel(sample_size=spec.sample_size, block_out_channels=spec.block_out_channels, attention_head_dim=spec.num_heads,
                             cross_attention_dim=spec.cross_attention_dim)
    u.load_state_dict(sd)
    return u.to(DEV).requires_grad_(False).eval()


def copy_lora(group, lora):
    with torch.no_grad():
        for layer, entries in lora.items():
            group[layer].layer.W_down.copy_(entries[0].W_down)
            group[layer].layer.W_up.copy_(entries[0].W_up)


def cosine(name, got, want, bound):
    got, want = got.double(), want.double()
    cos = float(got @ want / (got.norm() * want.norm()))
    ratio = float(got.norm() / want.norm())
    measured(f"{name} update cosine", cos, bound, above=True)
    print(f"{name} update norm ratio {ratio:.4f}")
    assert 0.8 < ratio < 1.25


def lora_delta(group, before):
    return torch.cat([torch.cat([(b.layer.W_down - before[k][0]).flatten(), (b.layer.W_up - before[k][1]).flatten()]).cpu()
                      for k, b in group.plugin_dict.items()])


def lora_before(group):
    return {k: (b.layer.W_down.detach().clone(), b.layer.W_up.detach().clone()) for k, b in group.plugin_dict.items()}


def ref_delta(group, lora, before):
    return torch.cat([torch.cat([(lora[k][0].W_down.detach() - before[k][0].cpu()).flatten(),
                                 (lora[k][0].W_up.detach() - before[k][1].cpu()).flatten()]) for k in group.plugin_dict])


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("max_norm", [1e-3, 1e9])
def test_tiny_lora_lion_steps_match_reference_loop(use_graph, max_norm):
    """Three Lion steps of TINY attention LoRA, eager and graph replay, with a clip engaged at every step (1e-3) and never (1e9)."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, group = make_hcpdiff(unet, None, [{"lr": LR, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(group, lora)
    ref = L.use_lion(S.ReferenceLoop(sd, lora, spec, lr=LR, max_grad_norm=max_norm), weight_decay=WD)
    before = lora_before(group)
    step = LoraTrainStep(unet, groups, lr=LR, weight_decay=WD, optimizer="lion", max_grad_norm=max_norm, use_cuda_graph=use_graph)
    assert step.v is None and step.optimizer_state_bytes == 4 * step.flat.numel
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=400 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    assert int(step.step_count) == 3
    cosine(f"lora graph={use_graph} max_norm={max_norm}", lora_delta(group, before), ref_delta(group, lora, before), COS)


def test_tiny_full_finetune_lion_steps_match_reference_loop():
    """Three Lion graph steps of every TINY UNet parameter, with EMA."""
    spec = U.TINY
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    groups, lora = make_hcpdiff(unet, [{"lr": 1e-5, "layers": [""]}], None)
    assert lora.empty() and len(groups) == 1
    names = [n for n, _ in unet.named_parameters()]
    ref_sd = {k: v.clone() for k, v in sd.items()}
    ref = L.use_lion(S.ReferenceLoop(ref_sd, None, spec, lr=1e-5, train_base=names), weight_decay=WD)
    p0 = {n: p.detach().clone() for n, p in unet.named_parameters()}
    step = LoraTrainStep(unet, groups, lr=1e-5, weight_decay=WD, optimizer="lion", ema={"decay_max": 0.999})
    for it in range(3):
        lat, noise, t, ehs = U.synthetic_batch(4, spec, seed=300 + it)
        l_ref = ref.micro_step(lat, noise, t, ehs)
        l_prod = float(step.step(lat, noise, t, ehs).cpu())
        assert abs(l_prod - l_ref) < 2e-2 * abs(l_ref), (it, l_prod, l_ref)
    du_p = torch.cat([(p.detach() - p0[n]).flatten().cpu() for n, p in unet.named_parameters()])
    du_r = torch.cat([(ref_sd[n].detach() - sd[n]).flatten() for n in names])
    cosine("full fine-tune", du_p, du_r, COS)
    # EMA follows the moved parameters (ModelEMA at steps 1..3 reads the Lion step counter)
    ema = torch.cat([e.flatten() for e in step.ema_state().values()]).cpu()
    assert not torch.equal(ema, torch.cat([p0[n].flatten() for n in names]).cpu())


def test_joint_te_unet_lion_steps_match_reference_loop():
    """Three Lion steps of the TINY UNet + a two-layer text encoder, both adapter sets in their own groups, clip_skip 1: the last
    layer's adapters get a zero gradient, so m stays 0, c = 0 and they only decay, as in the reference."""
    spec, tspec = U.TINY, CR.TINY_TE
    sd = U.init_params(spec)
    unet = tiny_unet(sd)
    ugroups, ugroup = make_hcpdiff(unet, None, [{"lr": 1e-4, "rank": 4, "alpha": 1.0, "layers": [r"re:.*\.attn.?$"]}])
    lora = U.init_lora(spec, rank=4)
    copy_lora(ugroup, lora)
    tsd = CR.init_params(tspec, seed=5)
    te = CLIPTextModel(**tspec.kwargs())
    te.load_state_dict(tsd)
    te = te.to(DEV).requires_grad_(False)
    tgroups, tgroup = make_hcpdiff(te, None, [{"lr": 1e-5, "rank": 4, "layers": [r"re:.*self_attn$", r"re:.*mlp$"]}], default_lr=1e-5)
    tlora = CR.init_lora(tspec, rank=4)
    copy_lora(tgroup, tlora)
    opts = {"n_repeats": 1, "clip_skip": 1, "clip_final_norm": True}
    step = LoraTrainStep(unet, ugroups + tgroups, lr=1e-4, weight_decay=WD, optimizer="lion", text_encoder=te, text_encoder_opts=opts)
    ref = L.use_lion(CR.joint_reference_loop(sd, lora, spec, tsd, tlora, tspec, opts, lr=1e-4, te_lr=1e-5), weight_decay=WD)
    before_u, before_t = lora_before(ugroup), lora_before(tgroup)
    for i in range(3):
        lat, noise, t, _ = U.synthetic_batch(2, spec, seed=100 + i)
        ids = CR.synthetic_ids(2, 1, seed=200 + i)
        loss = float(step.step(lat, noise, t, ids).cpu())
        loss_ref = ref.micro_step(lat, noise, t, ids)
        assert abs(loss - loss_ref) <= 2e-2 * abs(loss_ref), (i, loss, loss_ref)
    cosine("joint unet", lora_delta(ugroup, before_u), ref_delta(ugroup, lora, before_u), COS)
    live = [k for k in tgroup.plugin_dict if ".layers.1." not in k]
    got = torch.cat([torch.cat([(tgroup[k].layer.W_down - before_t[k][0]).flatten(), (tgroup[k].layer.W_up - before_t[k][1]).flatten()])
                     for k in live]).cpu()
    want = torch.cat([torch.cat([(tlora[k][0].W_down.detach() - before_t[k][0].cpu()).flatten(),
                                 (tlora[k][0].W_up.detach() - before_t[k][1].cpu()).flatten()]) for k in live])
    cosine("joint te", got, want, COS)
    # the skipped layer's adapters: p (1 - lr wd) rounded, three times, bit for bit as the reference
    skipped = [k for k in tgroup.plugin_dict if ".layers.1." in k]
    assert skipped
    for k in skipped:
        for got_p, ref_p, b0 in ((tgroup[k].layer.W_down, tlora[k][0].W_down, before_t[k][0]),
                                 (tgroup[k].layer.W_up, tlora[k][0].W_up, before_t[k][1])):
            assert not torch.equal(got_p, b0), f"{k}: not decayed"
            assert torch.equal(got_p.detach().cpu(), ref_p.detach()), k


LION_CFG = """
model:
  unet:
    _target_: hcp_diffusion_b200.models.UNet2DConditionModel
    sample_size: 16
    block_out_channels: [64, 128, 128, 128]
    attention_head_dim: 2
    cross_attention_dim: 64
  ema: {decay_max: 0.99}
"""


def test_train_ac_ft_lion_yaml_tiny_saves_and_resumes(tmp_path):
    """The entrypoint on cfgs/train/ft_lion_sd15_synthetic.yaml with a TINY UNet: trains with a finite loss, saves the full UNet
    and resumes from it."""
    import yaml
    from hcp_diffusion_b200.ckpt_manager import CkptManagerSafe
    from hcp_diffusion_b200.train_ac import Trainer
    from hcp_diffusion_b200.utils.config import load_config_with_cli
    with open(os.path.join(ROOT, "cfgs", "train", "ft_lion_sd15_synthetic.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"].update(yaml.safe_load(LION_CFG)["model"])
    cfg["exp_dir"] = str(tmp_path / "exp")
    cfg["train"].update(train_steps=3, save_step=3, log_step=1)
    cfg["data"].update(batch_size=2, num_samples=4)
    path = tmp_path / "ft_lion_tiny.yaml"
    path.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, "-m", "hcp_diffusion_b200.train_ac", "--cfg", str(path)], cwd=ROOT, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    last = [ln for ln in r.stdout.splitlines() if ln.startswith("step 3/3")]
    assert last and math.isfinite(float(last[0].split("loss")[1].split()[0])), r.stdout
    ck = str(tmp_path / "exp" / "ckpts" / "unet-3.safetensors")
    sd = CkptManagerSafe().load_ckpt(ck)
    assert "base" in sd and "base_ema" in sd
    conf = load_config_with_cli(str(path), [f"train.resume.ckpt_path.unet=[{ck}]", "train.resume.start_step=3", "train.train_steps=4"])
    tr = Trainer(conf)
    assert tr.step_fn.optimizer == "lion" and tr.step_fn.betas == (0.9, 0.99)
    assert float(tr.step_fn.segments[0]["hyper"][4]) == pytest.approx(1e-2)
    live = dict(tr.unet.named_parameters())
    for k, v in sd["base"].items():
        torch.testing.assert_close(live[k].detach().cpu(), v, msg=k, rtol=0, atol=0)
    tr.train()
