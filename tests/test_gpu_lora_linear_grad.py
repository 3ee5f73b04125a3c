"""GPU tests of the linear LoRA factor gradients at their planning edges (`pytest -m gpu`): hcp_lora_grad_pair (dW_down and dW_up of
one LoRA group in one launch of two independent problems) and hcp_lora_grad (one problem: each further input of a concatenated
layer, or any block table), as FusedLinearFn._lora_grads issues them for every adapted Linear and 1x1 Conv2d.

Each call goes straight through the C ABI and is compared with a float64 reference computed from the bf16 operands it reads
(tests/kernel_check.py, bound F32SUM; for CTAs that chain more than 6 128-row tiles in one accumulator, F32SUM scaled by the chain):

    dW_down[j, k] = scale * sum_m U[m, c0 + j] x[m, k]          dW_up[o, j] = alpha * sum_m dY[m, o0 + o] T[m, c0 + j]

Every destination lives in an fp32 canary buffer prefilled with 0.5: the kernels accumulate, and nothing outside the destinations
may change.  Columns of T / U that no block owns, and columns of x / dY outside every block's [n_lo, n_hi) (row padding included),
hold bf16 NaN, so a result that reads them is not finite.  The host-side planners are restated in tests/lora_linear_plan.py; each
case re-plans with the live SM count and asserts the branch it was chosen for.  The kernels reduce with fp32 atomics, so repeats are
not bit-identical and are not compared bit for bit.
"""
import pytest
import torch

from kernel_check import Canary, compare, f32sum_chain
from lora_linear_plan import TWO_INPUT_CASES, branches, grad_cases, grad_plan, lora_layout, pair_cases, pair_plan, slabs

pytestmark = pytest.mark.gpu

from hcp_diffusion_b200 import _lib  # noqa: E402
from hcp_diffusion_b200._lib import HcpError, LoraGradBlock, call, stream_ptr  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
NAN = float("nan")


def rnd(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV).to(BF)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def poison_columns(t, keep):
    """NaN in every column of t [M, ld] outside the [lo, hi) ranges of `keep`."""
    mask = torch.ones(t.shape[1], dtype=torch.bool, device=DEV)
    for lo, hi in keep:
        mask[lo:hi] = False
    t[:, mask] = NAN
    return t


def flat_canary(sizes):
    """One fp32 canary holding destinations of `sizes` elements back to back, prefilled with 0.5 -> (canary, offsets)."""
    offs = [sum(sizes[:i]) for i in range(len(sizes))]
    c = Canary(1, sum(sizes), dtype=F32)
    c.view.fill_(0.5)
    return c, offs


def table(entries):
    """entries: (n_lo, n_hi, c0, rank, scale, transpose_out, dst pointer, dst_ld) -> LoraGradBlock array."""
    arr = (LoraGradBlock * len(entries))()
    for a, (lo, hi, c0, r, s, tr, dst, ld) in zip(arr, entries):
        a.n_lo, a.n_hi, a.c0, a.rank, a.scale, a.transpose_out, a.dst, a.dst_ld = lo, hi, c0, r, s, tr, dst, ld
    return arr


# ----------------------------------------------------------------------------------------------------------------------------------
# a LoRA group: blocks (rank, o0, out_dim) over inputs x_i [M, K_i], issued as FusedLinearFn._lora_grads issues them
# ----------------------------------------------------------------------------------------------------------------------------------
class Group:
    def __init__(self, M, Ks, N, blocks, seed=0, pad=16):
        self.M, self.Ks, self.N, self.blocks = M, list(Ks), N, blocks
        self.ranks = [r for r, _, _ in blocks]
        self.c0s, _, self.R = lora_layout(self.ranks)
        self.K = sum(Ks)
        self.lds = self.R + 8
        owned = [(c0, c0 + r) for c0, r in zip(self.c0s, self.ranks)]
        self.U = poison_columns(rnd(M, self.lds, seed=seed + 1), owned)
        self.T = poison_columns(rnd(M, self.lds, seed=seed + 2), owned)
        # row pitches wider than the operands: the padding is NaN, and so are dY's columns of no block
        self.xs = [poison_columns(rnd(M, k + pad, seed=seed + 3 + i), [(0, k)]) for i, k in enumerate(Ks)]
        self.dy = poison_columns(rnd(M, N + pad, seed=seed + 10), [(o0, o0 + out) for _, o0, out in blocks])
        self.sd = [1.0 if i % 2 == 0 else 0.5 for i in range(len(blocks))]
        self.alpha = [0.75 / (i + 1) for i in range(len(blocks))]
        self.down, self.doff = flat_canary([r * self.K for r in self.ranks])
        self.up, self.uoff = flat_canary([out * r for r, _, out in blocks])

    def chunks(self):
        for q, pieces in slabs(self.ranks):
            for p0 in range(0, len(pieces), 8):
                yield q, pieces[p0:p0 + 8]

    def up_table(self, chunk):
        base = self.up.view.data_ptr()
        return table([(o0, o0 + out, cs, rows, self.alpha[i], 1, base + 4 * (self.uoff[i] + j0), r)
                      for i, j0, rows, cs in chunk for r, o0, out in [self.blocks[i]]])

    def down_table(self, chunk, koff, k):
        base = self.down.view.data_ptr()
        return table([(0, k, cs, rows, self.sd[i], 0, base + 4 * (self.doff[i] + j0 * self.K + koff), self.K) for i, j0, rows, cs in chunk])

    def run(self, pair=True):
        """pair: the pair launch on input 0 and hcp_lora_grad on the others (as _lora_grads); else every problem on its own.  Records
        the longest chain of 128-row tiles one CTA accumulates for each factor (its bound)."""
        n = sms()
        if pair:
            p = pair_plan(self.M, self.Ks[0], self.N, n)
            self.chain = {"down": p["down"]["tiles_per_cta"], "up": p["up"]["tiles_per_cta"]}
        else:
            self.chain = {"down": grad_plan(self.M, 0, self.Ks[0], n)["tiles_per_cta"],
                          "up": grad_plan(self.M, 0, self.N, n)["tiles_per_cta"]}
        for k in self.Ks[1:]:
            self.chain["down"] = max(self.chain["down"], grad_plan(self.M, 0, k, n)["tiles_per_cta"])
        launches = 0
        for q, chunk in self.chunks():
            Uq, Tq, nb = self.U.data_ptr() + 2 * 64 * q, self.T.data_ptr() + 2 * 64 * q, len(chunk)
            up = self.up_table(chunk)
            if not pair:
                call("hcp_lora_grad", Tq, self.lds, self.dy.data_ptr(), self.dy.shape[1], self.M, 0, self.N, up, nb, stream_ptr())
                launches += 1
            koff = 0
            for xi, (x, k) in enumerate(zip(self.xs, self.Ks)):
                down = self.down_table(chunk, koff, k)
                if xi == 0 and pair:
                    call("hcp_lora_grad_pair", Uq, x.data_ptr(), x.shape[1], k, down, Tq, self.dy.data_ptr(), self.dy.shape[1], self.N, up,
                         nb, self.M, self.lds, stream_ptr())
                else:
                    call("hcp_lora_grad", Uq, self.lds, x.data_ptr(), x.shape[1], self.M, 0, k, down, nb, stream_ptr())
                launches += 1
                koff += k
        torch.cuda.synchronize()
        return launches

    def results(self):
        """-> [(dW_down [r, K], dW_up [out, r])] of every block, the 0.5 prefill taken off."""
        d, u = self.down.view[0] - 0.5, self.up.view[0] - 0.5
        return [(d[self.doff[i]:self.doff[i] + r * self.K].view(r, self.K), u[self.uoff[i]:self.uoff[i] + out * r].view(out, r))
                for i, (r, _, out) in enumerate(self.blocks)]

    def check(self, name):
        x = torch.cat([x[:, :k] for x, k in zip(self.xs, self.Ks)], 1).to(F64)
        for i, ((r, o0, out), c0, (gd, gu)) in enumerate(zip(self.blocks, self.c0s, self.results())):
            compare(f"{name} dW_down[{i}] chain {self.chain['down']}", gd, self.sd[i] * (self.U[:, c0:c0 + r].to(F64).t() @ x),
                    f32sum_chain(self.chain["down"]), block=(64, 128))
            compare(f"{name} dW_up[{i}] chain {self.chain['up']}", gu,
                    self.alpha[i] * (self.dy[:, o0:o0 + out].to(F64).t() @ self.T[:, c0:c0 + r].to(F64)), f32sum_chain(self.chain["up"]),
                    block=(128, 64))
        self.down.check(f"{name} dW_down")
        self.up.check(f"{name} dW_up")


def pair_case_id(c):
    return c[0]


@pytest.mark.parametrize("case", pair_cases(), ids=pair_case_id)
def test_lora_grad_pair(case):
    """One LoRA group through hcp_lora_grad_pair, slab by slab and at most 8 pieces per launch."""
    name = case[0]
    _, M, K, N, blocks, want = next(c for c in pair_cases(sms()) if c[0] == name)
    p = pair_plan(M, K, N, sms())
    assert branches(want, p) == want, f"{name}: the planner at {sms()} SMs takes {branches(want, p)}, not {want}"
    g = Group(M, [K], N, blocks, seed=len(name))
    launches = g.run()
    g.check(f"pair {name} M{M} K{K} N{N} t0 {p['t0']} ({p['clamp']}) down {p['down']['n_tiles']}x{p['down']['splits']} "
            f"up {p['up']['n_tiles']}x{p['up']['splits']} launches {launches}")


@pytest.mark.parametrize("name", ["sd15_qkv", "r40x3", "uneven", "t0_low", "t0_high"])
def test_pair_matches_two_single_launches(name):
    """The pair launch against the same two problems issued as two hcp_lora_grad calls, within the bound of each other (and of the
    float64 reference); `uneven` gives dW_down 1 chunk against dW_up's 80, the clamped cases 1 or sms - 1 CTAs to one problem.
    The two runs chain different numbers of tiles per CTA: the difference is bounded by the longer chain."""
    _, M, K, N, blocks, _ = next(c for c in pair_cases(sms()) if c[0] == name)
    a, b = Group(M, [K], N, blocks, seed=7), Group(M, [K], N, blocks, seed=7)
    a.run(pair=True)
    b.run(pair=False)
    b.check(f"single launches {name}")
    tol = {f: f32sum_chain(max(a.chain[f], b.chain[f])) for f in ("down", "up")}
    for i, ((ad, au), (bd, bu)) in enumerate(zip(a.results(), b.results())):
        compare(f"pair vs single {name} dW_down[{i}]", ad, bd.to(F64), tol["down"], block=(64, 128))
        compare(f"pair vs single {name} dW_up[{i}]", au, bu.to(F64), tol["up"], block=(128, 64))


@pytest.mark.parametrize("M,K0,K1,N,blocks", TWO_INPUT_CASES)
def test_two_input_layer(M, K0, K1, N, blocks):
    """A layer over [x0 | x1] (an up block's conv_shortcut): the pair on x0, hcp_lora_grad on x1 into the columns K0.. of dW_down."""
    g = Group(M, [K0, K1], N, blocks, seed=3)
    launches = g.run()
    g.check(f"two inputs M{M} [{K0} | {K1}] -> {N} ranks {g.ranks} launches {launches}")


# ----------------------------------------------------------------------------------------------------------------------------------
# hcp_lora_grad with an arbitrary table
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", grad_cases(), ids=pair_case_id)
def test_lora_grad_table(case):
    """D[n, j] = scale * sum_m X[m, n] S[m, c0 + j] for n in [n_lo, n_hi) of every block, into dst[j, n - n_lo] (transpose_out = 0,
    dst_ld = n_hi - n_lo) or dst[n - n_lo, j] (transpose_out = 1, dst_ld = rank); X columns of no block and before n_begin are NaN."""
    name = case[0]
    _, M, n_begin, n_end, ldx, blocks, want = next(c for c in grad_cases(sms()) if c[0] == name)
    p = grad_plan(M, n_begin, n_end, sms())
    assert branches(want, p) == want, f"{name}: the planner at {sms()} SMs takes {branches(want, p)}, not {want}"
    ranks = [r for r, *_ in blocks]
    c0s, _, R = lora_layout(ranks)
    assert R == 64
    S = poison_columns(rnd(M, 72, seed=1), [(c0, c0 + r) for c0, r in zip(c0s, ranks)])
    X = poison_columns(rnd(M, ldx, seed=2), [(lo, hi) for _, lo, hi, _ in blocks])
    scales = [0.75 / (i + 1) for i in range(len(blocks))]
    dst, offs = flat_canary([r * (hi - lo) for r, lo, hi, _ in blocks])
    base = dst.view.data_ptr()
    call("hcp_lora_grad", S.data_ptr(), 72, X.data_ptr(), ldx, M, n_begin, n_end,
         table([(lo, hi, c0, r, s, tr, base + 4 * o, r if tr else hi - lo) for (r, lo, hi, tr), c0, s, o in zip(blocks, c0s, scales, offs)]),
         len(blocks), stream_ptr())
    torch.cuda.synchronize()
    got = dst.view[0] - 0.5
    label = f"lora_grad {name} M{M} [{n_begin}, {n_end}) chunks {p['n_tiles']} splits {p['splits']}x{p['tiles_per_cta']}"
    tol = f32sum_chain(p["tiles_per_cta"])
    for i, ((r, lo, hi, tr), c0, s, o) in enumerate(zip(blocks, c0s, scales, offs)):
        ref = s * (X[:, lo:hi].to(F64).t() @ S[:, c0:c0 + r].to(F64))                # [n, j]
        g = got[o:o + r * (hi - lo)]
        if tr:
            compare(f"{label} block {i} (transposed)", g.view(hi - lo, r), ref, tol, block=(128, 64))
        else:
            compare(f"{label} block {i}", g.view(r, hi - lo), ref.t(), tol, block=(64, 128))
    dst.check(label)


# ----------------------------------------------------------------------------------------------------------------------------------
# clean rejection
# ----------------------------------------------------------------------------------------------------------------------------------
def test_lora_grad_arguments_rejected_before_any_launch():
    M, K, N = 256, 128, 192
    S = torch.zeros(M, 64, dtype=BF, device=DEV)
    x, dy = torch.zeros(M, K, dtype=BF, device=DEV), torch.zeros(M, N, dtype=BF, device=DEV)
    dst = torch.zeros(64 * 256, dtype=F32, device=DEV)

    def blocks(n=1, lo=0, hi=K, c0=0, rank=4, tr=0, ld=None, dst_ptr=None):
        ld = ld if ld is not None else (rank if tr else hi - lo)
        return table([(lo, hi, c0, rank, 1.0, tr, dst.data_ptr() if dst_ptr is None else dst_ptr, ld)] * max(n, 1))

    def grad(nb=1, lds=64, ldx=K, m=M, n_begin=0, n_end=K, **kw):
        call("hcp_lora_grad", S.data_ptr(), lds, x.data_ptr(), ldx, m, n_begin, n_end, blocks(nb, **kw), nb, stream_ptr())

    def pair(nb=1, m=M, ldx=K, k=K, down=None, up=None):
        down = down or blocks(nb)
        up = up or blocks(nb, hi=N, tr=1)
        call("hcp_lora_grad_pair", S.data_ptr(), x.data_ptr(), ldx, k, down, S.data_ptr(), dy.data_ptr(), N, N, up, nb, m, 64, stream_ptr())

    torch.cuda.synchronize()
    before = _lib.launch_count
    cases = [
        ("1..8 blocks", lambda: grad(nb=0)),
        ("1..8 blocks", lambda: grad(nb=9)),
        ("1..8 blocks", lambda: pair(nb=9)),
        ("block descriptor", lambda: grad(rank=0)),
        ("block descriptor", lambda: grad(c0=61, rank=4)),                  # c0 + rank > 64
        ("block descriptor", lambda: grad(dst_ptr=0)),
        ("shape", lambda: grad(lds=56)),
        ("shape", lambda: grad(n_begin=-8)),
        ("shape", lambda: grad(n_begin=64, n_end=64, lo=64, hi=64)),
        ("lora_grad: M", lambda: grad(m=0)),
        ("lora_grad_pair: M", lambda: pair(m=-1)),
        ("block descriptor", lambda: pair(up=blocks(1, hi=N, tr=1, rank=0))),    # problem 1 only
        ("block descriptor", lambda: pair(up=blocks(1, hi=N, tr=1, c0=62))),
        ("block descriptor", lambda: pair(up=blocks(1, hi=N, tr=1, dst_ptr=0))),
        # X columns past the tensor map, block ranges outside the launch's columns, overlapping destination rows
        ("n_end > ldx", lambda: grad(ldx=120, n_end=128, hi=120)),
        ("n_end > ldx", lambda: pair(ldx=120, k=128, down=blocks(1, hi=120))),
        ("non-empty part", lambda: grad(lo=64, hi=64)),
        ("non-empty part", lambda: grad(lo=80, hi=64)),
        ("non-empty part", lambda: grad(n_begin=64, lo=56, hi=128)),
        ("non-empty part", lambda: grad(n_end=96, lo=0, hi=128)),
        ("non-empty part", lambda: pair(up=blocks(1, lo=0, hi=N + 8, tr=1))),    # problem 1 only
        ("non-empty part", lambda: pair(down=blocks(1, lo=0, hi=K + 8))),
        ("dst_ld below", lambda: grad(tr=1, rank=8, ld=7)),
        ("dst_ld below", lambda: grad(tr=0, lo=8, hi=128, ld=119)),
        ("dst_ld below", lambda: pair(up=blocks(1, hi=N, tr=1, rank=16, ld=8))),
    ]
    for match, fn in cases:
        with pytest.raises(HcpError, match=match):
            fn()
    torch.cuda.synchronize()
    assert _lib.launch_count == before
    # the boundaries themselves are accepted: dst_ld = rank / n_hi - n_lo, a block of the whole launch, n_end = ldx
    grad(tr=1, rank=8)
    grad(tr=0, lo=8, hi=128, n_begin=8)
    pair()
    torch.cuda.synchronize()
    assert _lib.launch_count == before + 3
