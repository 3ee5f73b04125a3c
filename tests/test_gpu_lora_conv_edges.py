"""GPU tests of the Conv2d LoRA (LoCon) and DreamArtist++ convolution path and of the LoRA operand packers at their tiling edges
(`pytest -m gpu`).

A LoCon block on a 3x3 convolution computes y = conv(x, W) + T . (alpha W_up)^T with T = conv3x3(x, W_down): the forward is the
convolution kernel with one more K-segment (the rank columns of T), dW_down is nine launches of the gradient kernel over the
shifted input boxes (one per tap), dW_up a plain gradient launch, and dX the input gradient plus a second convolution of
U = dY . (alpha W_up) through the taps of W_down accumulated in place.  The host-side planners these go through are restated in
tests/lora_conv_plan.py and the cases are chosen from it (tests/test_lora_conv_plan.py shows they reach every branch).  Each kernel is
called directly and compared with a float64 reference computed from the bf16 operands it reads (tests/kernel_check.py); every output
of a direct call lands in a canary buffer, and accumulated gradients start at 0.5.  The packers are checked bit for bit.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import F32SUM, FWD, LOCON, LORA, Canary, compare
from lora_conv_plan import CASES, DAPP_CASES, UP_CASES, conv_box, lora_grad_plan, lora_layout, slabs, split_plan, tile_n

pytestmark = pytest.mark.gpu

from hcp_diffusion_b200 import _lib, ops  # noqa: E402
from hcp_diffusion_b200._lib import HcpError, LoraGradBlock, LoraMergeJob, call, stream_ptr  # noqa: E402
from hcp_diffusion_b200.models import UNet2DConditionModel  # noqa: E402,F401  (runtime and models import each other: models first)
from hcp_diffusion_b200.ops import ConvLoraRef, ConvPack, LinearPack, LoraBlockRef  # noqa: E402
from hcp_diffusion_b200.runtime import pack_lora  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def case_id(c):
    return "B{}_{}x{}_{}-{}_s{}_r{}".format(*c[:6], "-".join(map(str, c[6])))


class Group:
    def __init__(self, pack):
        self.pack = pack


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == BF else torch.int32)


def conv_blocks(Cin, Cout, ranks, seed, branch=None, alpha=0.5):
    """fp32 W_down [r, Cin, 3, 3] / W_up [Cout, r, 1, 1] masters; the LoRA term is about as large as the host convolution's."""
    out = []
    for i, r in enumerate(ranks):
        down = rnd(r, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=seed + 2 * i, dtype=F32).requires_grad_(True)
        up = rnd(Cout, r, 1, 1, scale=1 / math.sqrt(r), seed=seed + 2 * i + 1, dtype=F32).requires_grad_(True)
        out.append(ConvLoraRef(down, up, alpha, branch))
    return out


def nchw(rows, B, H, W):
    return rows.reshape(B, H, W, -1).permute(0, 3, 1, 2)


def rows_of(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def conv_wgrad_ref(x, s_rows, B, H, W, stride):
    """float64 sum over pixels of S[m, j] x_shifted(kh, kw)[m, n] -> [j, n, 3, 3] (x [B*H*W, Cin], S [B*Ho*Wo, J])."""
    Ho, Wo = H // stride, W // stride
    Cin = x.shape[-1]
    xp = F.pad(x.to(F64).view(B, H, W, Cin), (0, 0, 1, 1, 1, 1))
    s = s_rows.to(F64)
    dw = torch.empty(s.shape[1], Cin, 3, 3, dtype=F64, device=x.device)
    for kh in range(3):
        for kw in range(3):
            dw[:, :, kh, kw] = s.t() @ xp[:, kh:kh + stride * Ho:stride, kw:kw + stride * Wo:stride].reshape(-1, Cin)
    return dw


def by_tap(dw):
    """[r, Cin, 3, 3] -> [9, r, Cin]: the gradient kernel's tiles (64 rank rows x 128 input channels of one tap) are 2-D blocks."""
    return dw.permute(2, 3, 0, 1).reshape(9, dw.shape[0], dw.shape[1])


# ----------------------------------------------------------------------------------------------------------------------------------
# packers, bit for bit
# ----------------------------------------------------------------------------------------------------------------------------------
def expect_conv_operands(pack):
    """The operands ConvPack's buffers must hold after pack_lora, arranged with torch from the same fp32 masters."""
    R, Cin, Cout = pack.R, pack.Cin, pack.Cout
    z = lambda *s: torch.zeros(s, dtype=BF, device=DEV)        # noqa: E731
    wt = {None: z(R, 3, 3, Cin), "n": z(R, 3, 3, Cin), "p": z(R, 3, 3, Cin)}
    blt = {None: z(R, Cout), "n": z(R, Cout), "p": z(R, Cout)}
    wdl, bl = z(Cin, 3, 3, R), z(Cout, R)
    for b in pack.lora:
        d = b.w_down.detach().to(BF)
        u = (b.alpha * b.w_up.detach()[:, :, 0, 0]).to(BF)
        cs = slice(b.c0, b.c0 + b.rank)
        wt[b.branch][cs] = d.permute(0, 2, 3, 1)
        wdl[..., cs] = (d.flip(2, 3) if pack.stride == 1 else d).permute(1, 2, 3, 0)
        bl[:, cs] = u
        blt[b.branch][cs] = u.t()
    return wt, wdl, bl, blt


def expect_linear_operands(pack):
    R, K, N = pack.R, pack.K, pack.N
    z = lambda *s: torch.zeros(s, dtype=BF, device=DEV)        # noqa: E731
    a = {None: z(R, K), "n": z(R, K), "p": z(R, K)}
    blt = {None: z(R, N), "n": z(R, N), "p": z(R, N)}
    at, bl = z(K, R), z(N, R)
    for b in pack.lora:
        d = b.w_down.detach().to(BF)
        u = (b.alpha * b.w_up.detach()).to(BF)
        cs, os_ = slice(b.c0, b.c0 + b.rank), slice(b.o0, b.o0 + b.out_dim)
        a[b.branch][cs] = d
        at[:, cs] = d.t()
        bl[os_, cs] = u
        blt[b.branch][cs, os_] = u.t()
    return a, at, bl, blt


def assert_bits(name, got, want):
    diff = int((bits(got) != bits(want)).sum())
    assert diff == 0, f"{name}: {diff} of {want.numel()} elements differ from the torch arrangement"


@pytest.mark.parametrize("dapp", [False, True])
@pytest.mark.parametrize("stride", [1, 2])
def test_conv_lora_packers_bit_exact(stride, dapp):
    """hcp_lora_pack_conv (flipped taps for stride 1, as-is for stride 2) and hcp_lora_pack's up-only jobs: ranks 40 | 24 fill the
    first slab, the third block starts the second (c0 64, R 128); Cout 72 is not a multiple of 64.  DreamArtist++: each block writes
    only its own branch's rows of W_down's forward taps and of BlT; the other branch's rows stay zero."""
    Cin, Cout, ranks = 64, 72, (40, 24, 40)
    pack = ConvPack(rnd(Cout, Cin, 3, 3, seed=1, dtype=F32), None, stride)
    branches = ("n", "p", "n") if dapp else (None,) * 3
    blocks = [blk for i, (r, br) in enumerate(zip(ranks, branches)) for blk in conv_blocks(Cin, Cout, (r,), 10 + 2 * i, br, alpha=0.3 + i)]
    pack.attach_lora(blocks)
    assert [b.c0 for b in blocks] == lora_layout(ranks)[0] == [0, 40, 64] and pack.R == 128
    pack_lora([Group(pack)])
    torch.cuda.synchronize()
    wt, wdl, bl, blt = expect_conv_operands(pack)
    if dapp:
        for br in ("n", "p"):
            assert_bits(f"Wt[{br}]", pack.Wt_br[br], wt[br])
            assert_bits(f"BlT[{br}]", pack.BlT_br[br], blt[br])
    else:
        assert_bits("Wt", pack.Wt, wt[None])
        assert_bits("BlT", pack.BlT, blt[None])
    assert_bits("Wdl", pack.Wdl, wdl)
    assert_bits("Bl", pack.Bl, bl)


@pytest.mark.parametrize("dapp", [False, True])
def test_linear_lora_pack_bit_exact(dapp):
    """hcp_lora_pack's linear jobs on a fused group of two hosts (out 72 each, K 200): a slab gap before the third block (c0 64),
    and with DreamArtist++ branches the row-masked A / BlT of each branch."""
    K, n = 200, 72
    pack = LinearPack(rnd(2 * n, K, seed=1, dtype=F32), None)
    spec = [(20, 0, "n"), (40, 0, "p"), (30, n, "n")]
    refs = []
    for i, (r, o0, br) in enumerate(spec):
        down = rnd(r, K, scale=0.1, seed=20 + 2 * i, dtype=F32)
        up = rnd(n, r, scale=0.3, seed=21 + 2 * i, dtype=F32)
        refs.append(LoraBlockRef(down, up, 0.25 * (i + 1), o0, br if dapp else None))
    pack.attach_lora(refs)
    assert [b.c0 for b in refs] == [0, 20, 64] and pack.R == 128
    pack_lora([Group(pack)])
    torch.cuda.synchronize()
    a, at, bl, blt = expect_linear_operands(pack)
    if dapp:
        for br in ("n", "p"):
            assert_bits(f"A[{br}]", pack.A_br[br], a[br])
            assert_bits(f"BlT[{br}]", pack.BlT_br[br], blt[br])
    else:
        assert_bits("A", pack.A, a[None])
        assert_bits("BlT", pack.BlT, blt[None])
    assert_bits("AT", pack.AT, at)
    assert_bits("Bl", pack.Bl, bl)


def ordered(t):
    """bf16 bit patterns as integers in value order (so that neighbouring bf16 values differ by one)."""
    b = t.view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


# merge jobs (o0, out_dim, ranks): four stacked blocks whose ranks sum to 64, out dims that are not multiples of 64
MERGE_JOBS = [(0, 72, (8, 16, 24, 16)), (72, 56, (20,)), (128, 24, (4, 12))]


@pytest.mark.parametrize("table", [True, False])
@pytest.mark.parametrize("tiled", [False, True])
def test_lora_merge_edges(tiled, table):
    """hcp_lora_merge on a fused group: W within one bf16 ulp of the correctly rounded float64 sum W_host + sum alpha W_up W_down
    (fp32 masters), WT exactly W^T, nothing outside the group's rows / columns written.  Row-major with in_dim 200 (a part-filled
    64-column tile) and three hosts (out_tot 152); k-block-major with in_dim 192 and the first two (out_tot 128).  Without a tile
    table the kernel finds each tile's job by binary search."""
    K = 192 if tiled else 200
    jobs_spec = MERGE_JOBS[:2] if tiled else MERGE_JOBS
    N = sum(out for _, out, _ in jobs_spec)
    g = torch.Generator().manual_seed(5)
    keep, jobs, tmap, tiles, want = [], [], [], 0, torch.zeros(N, K, dtype=F64, device=DEV)
    for i, (o0, out, ranks) in enumerate(jobs_spec):
        host = (torch.randn(out, K, generator=g) / math.sqrt(K)).to(DEV)
        j = LoraMergeJob()
        j.w_host, j.nblocks, j.in_dim, j.out_dim, j.o0, j.out_tot, j.tiled = host.data_ptr(), len(ranks), K, out, o0, N, int(tiled)
        acc = host.to(F64)
        for b, r in enumerate(ranks):
            down = (torch.randn(r, K, generator=g) / math.sqrt(K)).to(DEV)
            up = (torch.randn(out, r, generator=g) * 0.3).to(DEV)
            alpha = 0.5 / (b + 1)
            j.w_down[b], j.w_up[b], j.alpha[b], j.rank[b] = down.data_ptr(), up.data_ptr(), alpha, r
            acc = acc + alpha * (up.to(F64) @ down.to(F64))
            keep += [down, up]
        keep.append(host)
        want[o0:o0 + out] = acc
        j.tile0 = tiles
        n = -(-out // 64) * -(-K // 64)
        tmap += [i] * n
        tiles += n
        jobs.append(j)
    guard = 4096
    Wbuf = torch.zeros(N * K + guard, dtype=BF, device=DEV)
    WTbuf = torch.zeros(N * K + guard, dtype=BF, device=DEV)
    for j in jobs:
        j.W, j.WT = Wbuf.data_ptr(), WTbuf.data_ptr()
    dev = torch.frombuffer(bytearray(bytes((LoraMergeJob * len(jobs))(*jobs))), dtype=torch.uint8).to(DEV)
    tdev = torch.tensor(tmap, dtype=torch.int32, device=DEV) if table else None
    call("hcp_lora_merge", dev.data_ptr(), len(jobs), tiles, None if tdev is None else tdev.data_ptr(), 64, stream_ptr())
    torch.cuda.synchronize()
    assert not Wbuf[N * K:].any() and not WTbuf[N * K:].any(), "merge wrote past the operands"
    if tiled:
        W = Wbuf[:N * K].view(K // 64, N, 64).permute(1, 0, 2).reshape(N, K)
        WT = WTbuf[:N * K].view(N // 64, K, 64).permute(1, 0, 2).reshape(K, N)
    else:
        W, WT = Wbuf[:N * K].view(N, K), WTbuf[:N * K].view(K, N)
    ulps = (ordered(W) - ordered(want.to(BF))).abs()
    print(f"merge tiled={tiled} table={table}: {int((ulps == 1).sum())} of {ulps.numel()} elements one ulp from the rounded sum")
    assert int(ulps.max()) <= 1, f"merged weight {int(ulps.max())} bf16 ulps from the rounded float64 sum at {divmod(int(ulps.argmax()), K)}"
    assert torch.equal(bits(WT), bits(W.t())), "WT is not the exact transpose of W"


def test_lora_merge_rank_rows_at_edge_shape():
    """LinearPack.enable_merge with the rank rows riding the layer's own GEMMs at K 200, two hosts of 72 rows (o0 72): the rows past
    N of W hold W_down, the rows past K of WT hold (alpha W_up)^T in the host's columns and zeros in the other host's."""
    K, n = 200, 72
    g = torch.Generator().manual_seed(9)
    hosts = [(torch.randn(n, K, generator=g) / math.sqrt(K)).to(DEV) for _ in range(2)]
    pack = LinearPack(torch.cat(hosts), None)
    refs, per_host = [], []
    for i, ranks in enumerate(((8, 16, 24), (16,))):
        mine = [LoraBlockRef((torch.randn(r, K, generator=g) / math.sqrt(K)).to(DEV), (torch.randn(n, r, generator=g) * 0.3).to(DEV),
                             0.5, i * n) for r in ranks]
        refs += mine
        per_host.append((hosts[i], i * n, n, mine))
    pack.attach_lora(refs)
    assert pack.enable_merge(per_host) and pack.ext_rp == 64
    pack_lora([Group(pack)])
    torch.cuda.synchronize()
    N = 2 * n
    want = torch.cat([h.to(F64) + sum(b.alpha * (b.w_up.to(F64) @ b.w_down.to(F64)) for b in blocks) for h, _, _, blocks in per_host])
    assert int((ordered(pack.W[:N]) - ordered(want.to(BF))).abs().max()) <= 1
    assert torch.equal(bits(pack.WT[:K]), bits(pack.W[:N].t()))
    rows_w, rows_wt = torch.zeros(64, K, dtype=BF, device=DEV), torch.zeros(64, N, dtype=BF, device=DEV)
    for b in refs:
        rows_w[b.c0:b.c0 + b.rank] = b.w_down.to(BF)
        rows_wt[b.c0:b.c0 + b.rank, b.o0:b.o0 + n] = (b.alpha * b.w_up).to(BF).t()
    assert_bits("W rank rows", pack.W[N:], rows_w)
    assert_bits("WT rank rows", pack.WT[K:], rows_wt)


# ----------------------------------------------------------------------------------------------------------------------------------
# forward with the LoRA K-segment (hcp_conv3x3_bf16 with lora_t)
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_conv_lora_segment_forward(case, monkeypatch):
    """out = conv(x, W) + bias + rowbias + residual + T[:, :r] . Bl[:, :r]^T, row-major and (Cout % 64 == 0) k-block-major W.  The
    rank columns past r_tot hold 64.0 in T and Bl: the kernel must not read them.  Split-K equals the unsplit run and repeats bit
    for bit."""
    B, H, W, Cin, Cout, s, ranks = case
    _, r, R = lora_layout(ranks)
    sp = split_plan(B, H, W, Cin, Cout, s, R, r, sms())
    Ho, Wo = H // s, W // s
    M = B * Ho * Wo
    x = rnd(B, H * W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2, dtype=F32)
    bias = rnd(Cout, scale=0.5, seed=3, dtype=F32)
    rb = rnd(B, Cout + 8, scale=0.5, seed=4, dtype=F32)[:, 4:4 + Cout]
    res = rnd(M, Cout, seed=5)
    T = rnd(M, R, seed=6)
    Bl = rnd(Cout, R, scale=1 / math.sqrt(r), seed=7)
    T[:, r:], Bl[:, r:] = 64.0, 64.0
    pack = ConvPack(w, bias, s)
    yr = F.conv2d(nchw(x.to(F64), B, H, W), w.to(BF).to(F64), bias.to(F64), stride=s, padding=1) + rb.to(F64)[:, :, None, None]
    ref = rows_of(yr) + res.to(F64) + T[:, :r].to(F64) @ Bl[:, :r].to(F64).t()
    name = f"conv+lora {case_id(case)} splits {sp['splits']} (LoRA in split {sp['lora_split']})"
    lib = _lib.lib()
    assert lib.hcp_splitk_workspace_bytes(M, Cout, 9 * Cin + R) == (sp["splits"] * M * Cout * 4 if sp["splits"] > 1 else 0)

    def run(wop, tiled):
        out = Canary(M, Cout, ld=Cout, col0=0)
        ops.conv3x3_raw(x, wop, B, H, W, Cin, Cout, s, 0, out.view, bias=pack.bias, rowbias=rb, residual=res, rowbias_ld=rb.stride(0),
                        lora=(T, Bl, r, R), w_tiled=tiled)
        out.check(name)
        return out.view

    out = run(pack.W, False)
    compare(name, out, ref, FWD, block=(128, tile_n(Cout)))
    assert torch.equal(bits(run(pack.W, False)), bits(out)), f"{name}: a repeated call changed the result"
    if Cout % 64 == 0:
        pack.tile_weights()
        compare(f"{name} w_tiled", run(pack.W, True), ref, FWD, block=(128, tile_n(Cout)))
    if sp["splits"] > 1:
        monkeypatch.setattr(lib, "hcp_splitk_workspace_bytes", lambda *a: 0)          # no workspace: the same convolution unsplit
        whole = run(pack.W, pack.tiled)
        compare(f"{name} vs unsplit", out, whole.to(F64), FWD, block=(128, tile_n(Cout)))


# ----------------------------------------------------------------------------------------------------------------------------------
# factor gradients: dW_down (hcp_lora_grad_conv3x3) and dW_up (hcp_lora_grad, transpose_out = 1)
# ----------------------------------------------------------------------------------------------------------------------------------
def grad_blocks(pieces, ranks, offsets, base, scales, transpose_out=False, n=0):
    arr = (LoraGradBlock * len(pieces))()
    for k, (i, j0, rows, cs) in enumerate(pieces):
        arr[k].c0, arr[k].rank, arr[k].scale = cs, rows, scales[i]
        if transpose_out:                                       # dW_up [n, rank]: column j0 of block i
            arr[k].n_lo, arr[k].n_hi, arr[k].transpose_out, arr[k].dst_ld = 0, n, 1, ranks[i]
            arr[k].dst = base + 4 * (offsets[i] + j0)
        else:                                                   # dW_down [rank, Cin, 3, 3]: row j0 of block i
            arr[k].dst = base + 4 * (offsets[i] + j0 * n)
    return arr


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_lora_grad_conv3x3_dw_down(case):
    """dW_down[j, n, kh, kw] += scale * sum_m U[m, c0 + j] x_shifted(kh, kw)[m, n] for every block, slab by slab and at most 8 pieces
    per launch as Conv3x3Fn.backward issues them, from a U whose row pitch (R + 8) is wider than its rank columns."""
    B, H, W, Cin, Cout, s, ranks = case
    c0s, _, R = lora_layout(ranks)
    box, g = conv_box(B, H, W, s), lora_grad_plan(B, H, W, Cin, s, sms())
    M = B * (H // s) * (W // s)
    x = rnd(B * H * W, Cin, seed=1)
    U = rnd(M, R + 8, seed=2)
    scales = [1.0 if i % 2 == 0 else 0.5 for i in range(len(ranks))]
    offsets = [sum(r * Cin * 9 for r in ranks[:i]) for i in range(len(ranks))]
    dst = Canary(1, sum(ranks) * Cin * 9, dtype=F32)
    dst.view.fill_(0.5)
    launches = 0
    for q, pieces in slabs(ranks):
        for p0 in range(0, len(pieces), 8):
            chunk = pieces[p0:p0 + 8]
            arr = grad_blocks(chunk, ranks, offsets, dst.view.data_ptr(), scales, n=Cin * 9)
            call("hcp_lora_grad_conv3x3", U.data_ptr() + 2 * 64 * q, R + 8, x.data_ptr(), B, H, W, Cin, s, arr, len(chunk), stream_ptr())
            launches += 1
    ref = conv_wgrad_ref(x, U[:, :R], B, H, W, s)
    name = (f"dW_down {case_id(case)} box {box['bw']}x{box['bh']}x{box['bnimg']} chunks {g['col_chunks']} "
            f"splits {g['splits']}x{g['tiles_per_cta']} launches {launches}")
    got = dst.view[0] - 0.5
    for i, (c0, r) in enumerate(zip(c0s, ranks)):
        compare(f"{name} block {i}", by_tap(got[offsets[i]:offsets[i] + r * Cin * 9].view(r, Cin, 3, 3)),
                by_tap(scales[i] * ref[c0:c0 + r]), F32SUM, block=(64, 128))
    dst.check(name)


@pytest.mark.parametrize("M,N,ranks", UP_CASES)
def test_lora_grad_dw_up(M, N, ranks):
    """dW_up[o, j] += alpha * sum_m dY[m, o] T[m, c0 + j] (transpose_out = 1), over dY's 128-column chunks."""
    c0s, _, R = lora_layout(ranks)
    T, dy = rnd(M, R, seed=1), rnd(M, N, seed=2)
    alphas = [0.25 * (i + 1) for i in range(len(ranks))]
    offsets = [sum(r * N for r in ranks[:i]) for i in range(len(ranks))]
    dst = Canary(1, sum(ranks) * N, dtype=F32)
    dst.view.fill_(0.5)
    for q, pieces in slabs(ranks):
        for p0 in range(0, len(pieces), 8):
            chunk = pieces[p0:p0 + 8]
            arr = grad_blocks(chunk, ranks, offsets, dst.view.data_ptr(), alphas, transpose_out=True, n=N)
            call("hcp_lora_grad", T.data_ptr() + 2 * 64 * q, R, dy.data_ptr(), N, M, 0, N, arr, len(chunk), stream_ptr())
    ref = dy.to(F64).t() @ T.to(F64)
    got = dst.view[0] - 0.5
    for i, (c0, r) in enumerate(zip(c0s, ranks)):
        compare(f"dW_up M{M} N{N} ranks {ranks} block {i}", got[offsets[i]:offsets[i] + N * r].view(N, r), alphas[i] * ref[:, c0:c0 + r],
                F32SUM, block=(128, 64))
    dst.check("dW_up")


# ----------------------------------------------------------------------------------------------------------------------------------
# input gradient: dgrad through W plus the in-place dgrad through W_down
# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_conv_lora_dgrad(case):
    """dX = dgrad(dY, W) + dgrad(U, W_down) as Conv3x3Fn.backward computes it: the second convolution reads the packed taps of W_down
    (flipped at stride 1; at stride 2 four phase launches) and accumulates onto the first one's bf16 result in place."""
    B, H, W, Cin, Cout, s, ranks = case
    c0s, _, R = lora_layout(ranks)
    Ho, Wo = H // s, W // s
    M = B * Ho * Wo
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2, dtype=F32)
    pack = ConvPack(w, None, s)
    pack.attach_lora(conv_blocks(Cin, Cout, ranks, 10))
    pack_lora([Group(pack)])
    dy, U = rnd(M, Cout, seed=3), rnd(M, R, seed=4)
    dx = Canary(B * H * W, Cin, ld=Cin, col0=0)
    if s == 1:
        ops.conv3x3_raw(dy, pack.Wd, B, H, W, Cout, Cin, 1, 0, dx.view)
        ops.conv3x3_raw(U, pack.Wdl, B, H, W, R, Cin, 1, 0, dx.view, residual=dx.view)
    else:
        ops.conv3x3_raw(dy, pack.Wd, B, Ho, Wo, Cout, Cin, 2, 1, dx.view)
        ops.conv3x3_raw(U, pack.Wdl, B, Ho, Wo, R, Cin, 2, 1, dx.view, residual=dx.view)
    wdown = torch.zeros(R, Cin, 3, 3, dtype=F64, device=DEV)
    for b in pack.lora:
        wdown[b.c0:b.c0 + b.rank] = b.w_down.detach().to(BF).to(F64)
    xr = torch.zeros(B, Cin, H, W, dtype=F64, device=DEV, requires_grad=True)
    (F.conv2d(xr, w.to(BF).to(F64), stride=s, padding=1) * nchw(dy.to(F64), B, Ho, Wo)).sum().backward()
    g_main = xr.grad.clone()
    xr.grad = None
    (F.conv2d(xr, wdown, stride=s, padding=1) * nchw(U.to(F64), B, Ho, Wo)).sum().backward()
    compare(f"dX {case_id(case)}", dx.view, rows_of(g_main + xr.grad), LOCON, block=(128, tile_n(Cin)))
    dx.check("dX")


# ----------------------------------------------------------------------------------------------------------------------------------
# end to end through ops.conv3x3 / Conv3x3Fn, plain LoCon and DreamArtist++
# ----------------------------------------------------------------------------------------------------------------------------------
def check_end_to_end(B, H, W, Cin, Cout, s, blocks, name):
    """y, dX, d_rowbias and every block's dW_down / dW_up against float64 conv(x, W + sum alpha W_up x W_down) + bias + rowbias +
    residual; with DreamArtist++ branches the first half of the batch sees the 'n' blocks only, the second the 'p' blocks only."""
    Ho, Wo = H // s, W // s
    w = rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin), seed=2, dtype=F32)
    bias = rnd(Cout, scale=0.5, seed=3, dtype=F32)
    pack = ConvPack(w, bias, s)
    pack.attach_lora(blocks)
    pack.tile_weights()                                 # a frozen host: k-block-major when Cout % 64 == 0, as the runtime packs it
    pack_lora([Group(pack)])
    x = rnd(B, H * W, Cin, seed=1).requires_grad_(True)
    rb = rnd(B, Cout, scale=0.5, seed=4, dtype=F32).requires_grad_(True)
    res = rnd(B, Ho * Wo, Cout, seed=5)
    y = ops.conv3x3(pack, x, (B, H, W), rowbias=rb, residual=res)
    dy = rnd(B, Ho * Wo, Cout, seed=6)
    y.backward(dy)
    xr = nchw(x.detach().to(F64), B, H, W).requires_grad_(True)
    rbr = rb.detach().to(F64).requires_grad_(True)
    fac = [(b.w_down.detach().to(F64).requires_grad_(True), b.w_up.detach().to(F64).requires_grad_(True)) for b in blocks]
    halves = [("n", slice(0, B // 2)), ("p", slice(B // 2, B))] if pack.dapp else [(None, slice(0, B))]
    ys = []
    for br, sl in halves:
        weff = w.to(BF).to(F64)
        for b, (d_, u_) in zip(blocks, fac):
            if b.branch == br:
                weff = weff + b.alpha * torch.einsum("or,rikl->oikl", u_[:, :, 0, 0], d_)
        ys.append(F.conv2d(xr[sl], weff, bias.to(F64), stride=s, padding=1))
    yr = rows_of(torch.cat(ys) + rbr[:, :, None, None]).view(B, Ho * Wo, Cout) + res.to(F64)
    yr.backward(dy.to(F64))
    compare(f"{name} y", y.reshape(-1, Cout), yr.detach().reshape(-1, Cout), LOCON, block=(128, tile_n(Cout)))
    compare(f"{name} dX", x.grad.reshape(-1, Cin), rows_of(xr.grad), LOCON, block=(128, tile_n(Cin)))
    compare(f"{name} d_rowbias", rb.grad, rbr.grad, F32SUM)
    for i, (b, (d_, u_)) in enumerate(zip(blocks, fac)):
        compare(f"{name} dW_down[{i}] {b.branch or ''}", by_tap(b.w_down.grad), by_tap(d_.grad), LORA, block=(64, 128))
        compare(f"{name} dW_up[{i}] {b.branch or ''}", b.w_up.grad[:, :, 0, 0], u_.grad[:, :, 0, 0], LORA, block=(128, 64))


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_conv_lora_end_to_end(case):
    B, H, W, Cin, Cout, s, ranks = case
    check_end_to_end(B, H, W, Cin, Cout, s, conv_blocks(Cin, Cout, ranks, 10), f"locon {case_id(case)}")


@pytest.mark.parametrize("case", DAPP_CASES, ids=lambda c: "B{}_{}x{}_{}-{}_s{}".format(*c[:6]))
def test_dapp_conv_lora_end_to_end(case):
    B, H, W, Cin, Cout, s, rn, rp = case
    blocks = conv_blocks(Cin, Cout, rn, 10, "n") + conv_blocks(Cin, Cout, rp, 30, "p")
    check_end_to_end(B, H, W, Cin, Cout, s, blocks, f"dapp B{B} {H}x{W} {Cin}->{Cout} s{s}")


# ----------------------------------------------------------------------------------------------------------------------------------
# clean rejection
# ----------------------------------------------------------------------------------------------------------------------------------
def test_lora_conv_arguments_rejected_before_any_launch():
    x = torch.zeros(2, 16 * 16, 64, dtype=BF, device=DEV)
    w = torch.zeros(64, 3, 3, 64, dtype=BF, device=DEV)
    T, Bl = torch.zeros(2 * 256, 64, dtype=BF, device=DEV), torch.zeros(64, 64, dtype=BF, device=DEV)
    out = torch.empty(2 * 256 * 4, 64, dtype=BF, device=DEV)
    dpack = ConvPack(torch.zeros(64, 64, 3, 3, device=DEV), None, 1)
    dpack.attach_lora(conv_blocks(64, 64, (4,), 10, "n") + conv_blocks(64, 64, (4,), 20, "p"))
    pack_lora([Group(dpack)])
    dst = torch.zeros(64 * 64 * 9, dtype=F32, device=DEV)

    def blocks(n, c0=0, rank=4):
        arr = (LoraGradBlock * max(n, 1))()
        for b in arr:
            b.c0, b.rank, b.scale, b.dst = c0, rank, 1.0, dst.data_ptr()
        return arr

    def grad_conv(nb=1, c0=0, rank=4, Cin=64, H=16, W=16, stride=1):
        call("hcp_lora_grad_conv3x3", T.data_ptr(), 64, x.data_ptr(), 2, H, W, Cin, stride, blocks(nb, c0, rank), nb, stream_ptr())

    torch.cuda.synchronize()
    before = _lib.launch_count
    cases = [
        ("mode 0", lambda: ops.conv3x3_raw(x, w, 2, 16, 16, 64, 64, 2, 1, out, lora=(T, Bl, 4, 64))),       # mode 1 with lora_t
        ("LoRA segment", lambda: ops.conv3x3_raw(x, w, 2, 16, 16, 64, 64, 1, 0, out, lora=(T, Bl, 72, 64))),   # lora_r > lora_ld
        ("LoRA segment", lambda: ops.conv3x3_raw(x, w, 2, 16, 16, 64, 64, 1, 0, out, lora=(T, Bl, 4, 60))),    # lora_ld % 8 != 0
        ("arguments", lambda: grad_conv(nb=0)),
        ("arguments", lambda: grad_conv(nb=9)),
        ("block descriptor", lambda: grad_conv(c0=60, rank=8)),
        ("shape", lambda: grad_conv(Cin=96)),
        ("odd extent", lambda: grad_conv(H=15, stride=2)),
        ("W must divide 128", lambda: grad_conv(H=4, W=96)),
        ("even batch", lambda: ops.conv3x3(dpack, x[:1].expand(3, -1, -1).contiguous(), (3, 16, 16))),
    ]
    for match, fn in cases:
        with pytest.raises(HcpError, match=match):
            fn()
    torch.cuda.synchronize()
    assert _lib.launch_count == before
