"""Autograd wrappers around the C-ABI kernels (libhcpb200).

Every function here enqueues hand-written sm_90a kernels on the current CUDA stream through `_lib.call`; torch only
allocates the buffers and records the autograd graph.  Activations are bf16, "NHWC": a feature map [B,H,W,C] and the
token matrix [B*H*W, C] are the same memory.

Gradient fan-in is folded into producer kernels instead of separate adds: the normalisation functions return an alias of
their input next to the normalised output; the residual consumer uses the alias, so the normalisation backward receives
both gradients and adds them inside its own kernel.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import AttnArgs, AttnBwdArgs, ConvArgs, GemmArgs, GroupNormArgs, call, ptr, stream_ptr

BF16 = torch.bfloat16

# LoRA on Linear / 1x1 hosts whose adapters apply to every row: the adapters are MERGED into the bf16 weight operands once per step
# (W + sum alpha W_up W_down -- literally what the reference layer computes, lora_layers_patch.py:44-57), so the forward and the
# input gradient are plain GEMMs; the rank-r products T = x A^T / U = dY (alpha B) only feed the factor gradients, off the critical
# path.  HCP_LORA_MERGE=0 (or `ops.LORA_MERGE = False` before the packs are built) keeps the K-segment formulation, which DreamArtist++
# (per-branch adapters) always uses.
LORA_MERGE = os.environ.get("HCP_LORA_MERGE", "1") != "0"
# Frozen (and merged-LoRA) weight operands are stored K-BLOCK-MAJOR, [K/64][rows][64]: a TMA box of the B operand is then one
# contiguous run of 128 B x rows instead of `rows` 128-byte pieces at a 2K-byte pitch.  The small-M layers (16x16 / 8x8 levels) stream
# every weight byte from HBM exactly once per pass; whole-page reads are what lets them approach the HBM roofline.
WEIGHT_TILED = os.environ.get("HCP_WEIGHT_TILED", "0") != "0"
# Merged-LoRA layers carry their rank-r factors as extra rows of the weight operands, so T = x W_down^T and U = dY (alpha W_up) come
# out of the layer's own forward / dgrad GEMM as a second output (hcp_gemm_args.out2) instead of two skinny GEMM launches per layer.
LORA_EXT = os.environ.get("HCP_LORA_EXT", "1") != "0"


def tile_kmajor(w2d: torch.Tensor) -> torch.Tensor:
    """[rows, K] (K % 64 == 0) -> k-block-major [K/64, rows, 64], contiguous."""
    rows, K = w2d.shape
    return w2d.reshape(rows, K // 64, 64).permute(1, 0, 2).contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# side stream: work that is OFF the critical path of the step (LoRA-gradient kernels, the cross-attention k/v projections of the
# text embedding) is enqueued on a second stream so that it fills the SMs the small kernels of the main chain leave idle.
# Opt-in (LoraTrainStep turns it on and joins the stream before the optimizer); plain autograd users keep one stream.
# ----------------------------------------------------------------------------------------------------------------------
class _Side:
    enabled = False
    stream: Optional["torch.cuda.Stream"] = None
    used = False
    keep: list = []          # tensors the side stream reads: kept alive (no allocator reuse) until the join


def set_side_stream(on: bool) -> None:
    _Side.enabled = bool(on) and os.environ.get("HCP_SIDE_STREAM", "1") != "0"


def side_enabled() -> bool:
    return _Side.enabled


def fork_side(*keep: torch.Tensor) -> "torch.cuda.Stream":
    """Side stream, ordered after everything enqueued on the current stream so far."""
    if _Side.stream is None:
        _Side.stream = torch.cuda.Stream()
    _Side.stream.wait_stream(torch.cuda.current_stream())
    _Side.used = True
    _Side.keep.extend(t for t in keep if t is not None)
    return _Side.stream


def join_side() -> None:
    """The current stream waits for the side stream (call before anything consumes the LoRA gradients)."""
    if _Side.used:
        torch.cuda.current_stream().wait_stream(_Side.stream)
        _Side.used = False
    _Side.keep.clear()


# ----------------------------------------------------------------------------------------------------------------------
# dropout (reference: nn.Dropout on the whole output of a patched layer, hcpdiff/models/lora_base_patch.py:74).  The mask is a
# function of a device-resident (seed, draw) pair and a per-call `site` number: the backward pass regenerates it, CUDA-graph
# replays read the advanced `draw` and get fresh masks.
# ----------------------------------------------------------------------------------------------------------------------
class _Drop:
    state: Optional[torch.Tensor] = None     # int64 [2] on the device: (seed, draw)
    site = 0                                 # call sites of the current forward pass
    used = False


def set_dropout_seed(seed: int) -> None:
    dev = torch.device("cuda", torch.cuda.current_device())
    _Drop.state = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=dev)


def _dropout_state() -> torch.Tensor:
    if _Drop.state is None:
        set_dropout_seed(torch.initial_seed())
    return _Drop.state


def advance_dropout() -> None:
    """End of one forward/backward: the next one draws new masks (one tiny kernel, only when a dropout site ran)."""
    if _Drop.used and _Drop.state is not None:
        call("hcp_counter_add_u64", _Drop.state.data_ptr() + 8, 1, stream_ptr())
    _Drop.site = 0


def dropout_state_snapshot():
    return None if _Drop.state is None else _Drop.state.clone()


def dropout_state_restore(saved) -> None:
    if saved is not None and _Drop.state is not None:
        _Drop.state.copy_(saved)


class DropoutFn(torch.autograd.Function):
    """out[:, c0:c0+n] = dropout_p(y[:, c0:c0+n]) for every (c0, n, p) range (p = 0: copy), + residual + per-image row bias.
    y bf16 [..., N]; the ranges must tile [0, N)."""

    @staticmethod
    def forward(ctx, ranges, residual: Optional[torch.Tensor], rowbias: Optional[torch.Tensor], rows_per_group: int, y: torch.Tensor):
        y = _chk(y, "dropout input")
        N = y.shape[-1]
        M = y.numel() // N
        res = None if residual is None else _chk(residual, "dropout residual")
        out = torch.empty_like(y)
        st = _dropout_state()
        sites = []
        rb_ld = 0 if rowbias is None else rowbias.stride(0)
        for (c0, n, p) in ranges:
            _Drop.site += 1
            _Drop.used = True
            sites.append(_Drop.site)
            call("hcp_dropout_bf16", y.data_ptr() + 2 * c0, N, None if res is None else res.data_ptr() + 2 * c0, N,
                 None if rowbias is None else rowbias.data_ptr() + 4 * c0, rb_ld, max(rows_per_group, 1), M, n, float(p), st.data_ptr(),
                 sites[-1], out.data_ptr() + 2 * c0, N, stream_ptr())
        ctx.ranges, ctx.sites, ctx.has_res = list(ranges), sites, residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = _chk(dout, "dropout grad")
        N = dout.shape[-1]
        M = dout.numel() // N
        dy = torch.empty_like(dout)
        st = _dropout_state()
        for (c0, n, p), site in zip(ctx.ranges, ctx.sites):
            call("hcp_dropout_bf16", dout.data_ptr() + 2 * c0, N, None, 0, None, 0, 1, M, n, float(p), st.data_ptr(), site,
                 dy.data_ptr() + 2 * c0, N, stream_ptr())
        return None, (dout if (ctx.has_res and ctx.needs_input_grad[1]) else None), None, None, dy


def dropout_cols(y, ranges, residual=None, rowbias=None, rows_per_group=0):
    return DropoutFn.apply(tuple(ranges), residual, rowbias, rows_per_group, y)


# ----------------------------------------------------------------------------------------------------------------------
# gradient-ready notifications (full fine-tune, data parallel): the engine buckets the flat gradient buffer and all-reduces a bucket
# as soon as the kernels producing its last parameter gradient have been enqueued (the reference's DDP reducer hooks).
# ----------------------------------------------------------------------------------------------------------------------
class _GradHook:
    cb = None


def set_grad_ready_callback(cb) -> None:
    _GradHook.cb = cb


def notify_grad(*params) -> None:
    if _GradHook.cb is not None:
        _GradHook.cb([p for p in params if p is not None])


def _chk(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dtype != BF16 or not t.is_cuda:
        raise _lib.HcpError(f"{name}: expected a CUDA bf16 tensor, got {t.dtype} on {t.device}")
    return t if t.is_contiguous() else t.contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# raw launches
# ----------------------------------------------------------------------------------------------------------------------
def gemm_raw(a_list: Sequence[Tuple[torch.Tensor, int, int]], b_list: Sequence[Tuple[torch.Tensor, int, int, int]], M: int, N: int,
             out: torch.Tensor, ldo: int, bias: Optional[torch.Tensor] = None, rowbias: Optional[torch.Tensor] = None,
             rows_per_group: int = 0, residual: Optional[torch.Tensor] = None, ldr: int = 0,
             out2: Optional[torch.Tensor] = None, ldo2: int = 0, n_main: int = 0) -> None:
    """out[M,N] = sum_s A_s . B_s^T (+bias +rowbias +residual).
    a_list: (tensor_or_ptr_holder, lda, k);  b_list: (tensor, ldb, n_rows_b, elem_offset[, k_block_major]) -- for a k-block-major
    operand ldb is the row count of one k-block slab (see hcp_gemm_args.flags)."""
    g = GemmArgs()
    g.nseg = len(a_list)
    for s, ((a, lda, k), bent) in enumerate(zip(a_list, b_list)):
        b, ldb, nrb, boff = bent[:4]
        g.a[s] = a.data_ptr()
        g.lda[s] = lda
        g.k[s] = k
        g.b[s] = b.data_ptr() + 2 * boff
        g.ldb[s] = ldb
        g.n_rows_b[s] = nrb
        if len(bent) > 4 and bent[4]:
            g.flags |= 1 << s
    g.M, g.N = M, N
    g.bias = ptr(bias)
    g.rowbias = ptr(rowbias)
    g.rows_per_group = rows_per_group
    g.residual = ptr(residual)
    g.ldr = ldr
    g.out = out.data_ptr()
    g.ldo = ldo
    if out2 is not None:          # columns [n_main, N) -> out2 (hcp_gemm_args.out2)
        g.out2, g.ldo2, g.n_main = out2.data_ptr(), ldo2, n_main
    wsb = 0 if out2 is not None else _lib.lib().hcp_splitk_workspace_bytes(M, N, sum(k for _, _, k in a_list))
    if wsb:
        ws = torch.empty((wsb // 4,), dtype=torch.float32, device=out.device)
        g.workspace, g.workspace_bytes = ws.data_ptr(), wsb
    call("hcp_gemm_bf16", C.byref(g), stream_ptr())


def conv3x3_raw(x: torch.Tensor, w: torch.Tensor, B: int, Hin: int, Win: int, Cin: int, Cout: int, stride: int, mode: int,
                out: torch.Tensor, bias=None, rowbias=None, residual=None, rowbias_ld: int = 0, lora=None, w_tiled: bool = False) -> None:
    """`lora`: (T [M,R] bf16, Bl [Cout,R] bf16, r_used, R) -- the Conv2d-LoRA K-segment of a forward convolution."""
    a = ConvArgs()
    a.x, a.w = x.data_ptr(), w.data_ptr()
    a.B, a.Hin, a.Win, a.Cin, a.Cout = B, Hin, Win, Cin, Cout
    a.stride, a.mode = stride, mode
    a.w_tiled = int(w_tiled)
    a.bias, a.rowbias, a.residual = ptr(bias), ptr(rowbias), ptr(residual)
    a.rowbias_ld = rowbias_ld
    a.out = out.data_ptr()
    if lora is not None:
        a.lora_t, a.lora_b, a.lora_r, a.lora_ld = lora[0].data_ptr(), lora[1].data_ptr(), lora[2], lora[3]
    if mode == 0:
        Mo = B * (Hin // stride) * (Win // stride)
        wsb = _lib.lib().hcp_splitk_workspace_bytes(Mo, Cout, 9 * Cin + (lora[3] if lora is not None else 0))
        if wsb:
            ws = torch.empty((wsb // 4,), dtype=torch.float32, device=out.device)
            a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
    call("hcp_conv3x3_bf16", C.byref(a), stream_ptr())


# ----------------------------------------------------------------------------------------------------------------------
# packed weights
# ----------------------------------------------------------------------------------------------------------------------
class LoraBlockRef:
    """One LoRA block inside a fused linear group (see hcp_lora_job in include/hcp_b200.h).
    `branch`: None (applies to every row) or 'p' / 'n' -- DreamArtist++ adapters, reference DAPPPatchContainer.forward
    (hcpdiff/models/lora_layers_patch.py:102-133): the first half of the batch sees the 'n' blocks, the second half the 'p' blocks."""
    __slots__ = ("w_down", "w_up", "alpha", "rank", "in_dim", "out_dim", "c0", "o0", "g_down", "g_up", "branch")

    def __init__(self, w_down, w_up, alpha, o0, branch=None):
        self.w_down, self.w_up, self.alpha = w_down, w_up, float(alpha)
        self.rank, self.in_dim = w_down.shape[0], w_down.shape[1]     # Linear [r,in] or 1x1 Conv2d [r,in,1,1]
        self.out_dim = w_up.shape[0]
        self.c0, self.o0 = 0, o0
        self.branch = branch
        self.g_down = None   # optional fp32 views into a flat gradient buffer (direct accumulation)
        self.g_up = None


class LinearPack:
    """bf16 operands of one (possibly fused, possibly LoRA-patched) linear group  y = x . W^T + b.

    LoRA blocks of the group share R = 64-padded rank columns: T = x . A^T [M,R] is the extra K-segment of the main GEMM
    against alpha*W_up packed as Bl [N,R].  A block never straddles a 64-column slab unless its rank exceeds 64 (then it starts
    on a slab boundary), so the gradient kernel works slab by slab."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], k_splits: Optional[Sequence[int]] = None):
        # weight fp32/bf16 [N, K]
        self.N, self.K = weight.shape
        self.W = weight.detach().to(BF16).contiguous()
        self.WT = self.W.t().contiguous()
        # k-block-major operand layout (set by `tile_weights`, once the pack is known to hold frozen / merged weights only)
        self.tiled = False
        self.bias = None if bias is None else bias.detach().float().contiguous()
        self.k_splits = list(k_splits) if k_splits else [self.K]
        self.lora: List[LoraBlockRef] = []
        self.r_tot = 0          # rank columns in use (incl. alignment gaps)
        self.R = 0              # r_tot padded to a multiple of 64
        self.dapp = False
        self.A = self.AT = self.Bl = self.BlT = None
        self.A_br = self.BlT_br = None      # DAPP: {'n': ..., 'p': ...} row-masked variants of A / BlT
        # merged mode: [(fp32 host weight [n, K], first output row o0, n, [LoraBlockRef, ...])]; W / WT are then rewritten every step
        # by hcp_lora_merge (runtime.pack_lora) and the GEMMs carry no LoRA segment
        self.merged: List[Tuple[torch.Tensor, int, int, list]] = []
        # merged mode with rank columns riding the layer's own GEMMs: W is [N + ext_rp, K] with W_down in the extra rows (the forward
        # GEMM also emits T = x W_down^T), WT is [K + ext_rp, N] with alpha*W_up^T in the extra rows (the dgrad GEMM also emits U)
        self.ext_rp = 0
        # full fine-tune: [(weight Parameter [n, K] (or [n, K, 1, 1]), bias Parameter or None, first output row o0, n)] of the hosts
        # whose parameters are trained; their bf16 operands are refreshed from the fp32 masters every step (repack_jobs)
        self.train: List[Tuple[torch.Tensor, Optional[torch.Tensor], int, int]] = []

    def tile_weights(self) -> None:
        """W [N,K] -> [K/64][N][64], WT [K,N] -> [N/64][K][64] (frozen or merged weights only: hcp_repack_weights writes row-major)."""
        if self.tiled or self.train or self.ext_rp or self.K % 64 or self.N % 64 or any(k % 64 for k in self.k_splits):
            return
        self.W, self.WT = tile_kmajor(self.W), tile_kmajor(self.WT)
        self.tiled = True

    def b_fwd(self, off: int):
        """b_list entry of the forward operand for the input segment starting at column `off`."""
        if self.tiled:
            return (self.W, self.N, self.N, (off // 64) * self.N * 64, True)
        return (self.W, self.K, self.N, off)

    def b_dgrad(self, off: int, k: int):
        """b_list entry of W^T rows [off, off + k) (the dX GEMM of the input segment at column `off`)."""
        if self.tiled:
            return (self.WT, self.K, k, off * 64, True)
        return (self.WT, self.N, k, off * self.N)

    def repack_jobs(self) -> List[_lib.RepackJob]:
        out = []
        for w, b, o0, n in self.train:
            j = _lib.RepackJob()
            j.src, j.dst0, j.dst1 = w.data_ptr(), self.W.data_ptr(), self.WT.data_ptr()
            j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = 0, n, self.K, o0, self.N, 0
            out.append(j)
            if b is not None and self.bias is not None and b.requires_grad:
                j = _lib.RepackJob()
                j.src, j.dst0, j.dst1 = b.data_ptr(), self.bias.data_ptr(), None
                j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = 2, n, 1, o0, 0, 0
                out.append(j)
        return out

    def attach_lora(self, blocks: List[LoraBlockRef]) -> None:
        self.lora = blocks
        c = 0
        for b in blocks:
            if b.in_dim != self.K:
                raise _lib.HcpError(f"LoRA block input width {b.in_dim} does not match the layer ({self.K})")
            if b.rank > 64 or (c % 64) + b.rank > 64:
                c = (c + 63) // 64 * 64
            b.c0 = c
            c += b.rank
        self.r_tot = c
        self.R = (c + 63) // 64 * 64
        if self.R > 1024:
            raise _lib.HcpError(f"LoRA ranks of one fused linear group sum to {c} (> 1024 columns)")
        self.dapp = any(b.branch is not None for b in blocks)
        dev = self.W.device
        z = lambda *shape: torch.zeros(shape, dtype=BF16, device=dev)   # noqa: E731
        self.AT = z(self.K, self.R)
        self.Bl = z(self.N, self.R)
        if self.dapp:
            self.A_br = {"n": z(self.R, self.K), "p": z(self.R, self.K)}
            self.BlT_br = {"n": z(self.R, self.N), "p": z(self.R, self.N)}
            self.A = self.BlT = None
        else:
            self.A = z(self.R, self.K)
            self.BlT = z(self.R, self.N)

    def enable_merge(self, hosts: Sequence[Tuple[torch.Tensor, int, int, list]]) -> bool:
        """Switch the pack to merged weights if every patched host qualifies (fp32 master weight, <= 4 stacked blocks, ranks summing
        to <= 64, 8-element alignment); returns whether it did."""
        if self.dapp or self.train or not self.lora or self.K % 8 or self.N % 8:
            return False
        for w, o0, n, blocks in hosts:
            if w.dtype != torch.float32 or not w.is_contiguous() or len(blocks) > 4 or sum(b.rank for b in blocks) > 64 or o0 % 8 or n % 8:
                return False
        self.merged = [h for h in hosts if h[3]]
        if LORA_EXT and self.R == 64 and len(self.k_splits) == 1 and not self.tiled:
            rp = (self.r_tot + 7) // 8 * 8
            dev = self.W.device
            W = torch.zeros((self.N + rp, self.K), dtype=BF16, device=dev)
            WT = torch.zeros((self.K + rp, self.N), dtype=BF16, device=dev)
            W[:self.N].copy_(self.W)
            WT[:self.K].copy_(self.WT)
            self.W, self.WT, self.ext_rp = W, WT, rp
            self.A, self.BlT = W[self.N:], WT[self.K:]            # hcp_lora_pack writes the factors straight into the extra rows
        return True

    def merge_jobs(self) -> List[_lib.LoraMergeJob]:
        out = []
        for w, o0, n, blocks in self.merged:
            j = _lib.LoraMergeJob()
            j.w_host = w.data_ptr()
            for i, b in enumerate(blocks):
                j.w_down[i], j.w_up[i], j.alpha[i], j.rank[i] = b.w_down.data_ptr(), b.w_up.data_ptr(), b.alpha, b.rank
            j.nblocks, j.in_dim, j.out_dim, j.o0, j.out_tot = len(blocks), self.K, n, o0, self.N
            j.W, j.WT, j.tiled = self.W.data_ptr(), self.WT.data_ptr(), int(self.tiled)
            out.append(j)
        return out

    def jobs(self) -> List[_lib.LoraJob]:
        out = []
        for b in self.lora:
            branches = ([b.branch] if b.branch is not None else ["n", "p"]) if self.dapp else [None]
            for br in branches:
                j = _lib.LoraJob()
                j.w_down, j.w_up, j.alpha = b.w_down.data_ptr(), b.w_up.data_ptr(), b.alpha
                j.rank, j.in_dim, j.out_dim = b.rank, b.in_dim, b.out_dim
                j.c0, j.o0, j.out_tot, j.ld_r = b.c0, b.o0, self.N, self.R
                A, BlT = (self.A, self.BlT) if br is None else (self.A_br[br], self.BlT_br[br])
                j.A, j.AT, j.Bl, j.BlT = A.data_ptr(), self.AT.data_ptr(), self.Bl.data_ptr(), BlT.data_ptr()
                out.append(j)
        return out

    def slabs(self):
        """[(slab index, [(block, first rank row j0, rows, first column inside the slab)])] for the gradient kernel."""
        out = []
        for q in range(self.R // 64):
            lo, hi = 64 * q, 64 * q + 64
            pieces = []
            for b in self.lora:
                a, e = max(lo, b.c0), min(hi, b.c0 + b.rank)
                if a < e:
                    pieces.append((b, a - b.c0, e - a, a - lo))
            if pieces:
                out.append((q, pieces))
        return out


class ConvLoraRef:
    """One LoRA block on a 3x3 convolution (reference LoraLayer.Conv2dLayer, lora_layers_patch.py:64-100):
    W_down fp32 [r, Cin, 3, 3], W_up fp32 [Cout, r, 1, 1], alpha."""
    __slots__ = ("w_down", "w_up", "alpha", "rank", "c0", "branch")

    def __init__(self, w_down, w_up, alpha, branch=None):
        self.w_down, self.w_up, self.alpha = w_down, w_up, float(alpha)
        self.rank = w_down.shape[0]
        self.c0 = 0
        self.branch = branch       # None, or 'p' / 'n' (DreamArtist++: batch = [negative half | positive half])


class ConvPack:
    """bf16 operands of one 3x3 convolution (weights [Cout,Cin,3,3] fp32 -> tap-major K-major matrices), optionally with LoCon
    blocks: y = conv(x, W) + T . (alpha W_up)^T with T = conv3x3(x, W_down) -- the reference's conv(x, W + W_up x W_down)
    (lora_layers_patch.py:91-98) without materialising the [Cout,Cin,3,3] delta."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], stride: int):
        self.Cout, self.Cin = weight.shape[0], weight.shape[1]
        self.stride = stride
        w = weight.detach().to(BF16)
        self.W = w.permute(0, 2, 3, 1).contiguous()                          # [Cout, kh, kw, Cin]
        if stride == 1:
            self.Wd = w.flip(2, 3).permute(1, 2, 3, 0).contiguous()          # dgrad: [Cin, kh', kw', Cout], taps flipped
        else:
            self.Wd = w.permute(1, 2, 3, 0).contiguous()                     # stride-2 dgrad arrangement (not flipped)
        self.bias = None if bias is None else bias.detach().float().contiguous()
        self.lora: List[ConvLoraRef] = []
        self.r_tot = self.R = 0
        self.dapp = False
        self.train: Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]] = None     # (weight, bias) Parameters when the layer is trained
        self.Wt = self.Wdl = self.Bl = self.BlT = None
        self.Wt_br = self.BlT_br = None      # DAPP: {'n': ..., 'p': ...} row-masked variants of Wt / BlT
        self.tiled = False

    def tile_weights(self) -> None:
        """W [Cout, 9*Cin] / Wd [Cin, 9*Cout] -> k-block-major [9*C/64][rows][64] (frozen layers only)."""
        if self.tiled or self.train is not None or self.Cout % 64:
            return
        self.W = tile_kmajor(self.W.reshape(self.Cout, 9 * self.Cin))
        self.Wd = tile_kmajor(self.Wd.reshape(self.Cin, 9 * self.Cout))
        self.tiled = True

    def repack_jobs(self) -> List[_lib.RepackJob]:
        if self.train is None:
            return []
        w, b = self.train
        j = _lib.RepackJob()
        j.src, j.dst0, j.dst1 = w.data_ptr(), self.W.data_ptr(), self.Wd.data_ptr()
        j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = 1, self.Cout, self.Cin, 0, 0, 1 if self.stride == 1 else 0
        out = [j]
        if b is not None and self.bias is not None and b.requires_grad and b.data_ptr() != self.bias.data_ptr():
            j = _lib.RepackJob()
            j.src, j.dst0, j.dst1 = b.data_ptr(), self.bias.data_ptr(), None
            j.kind, j.rows, j.K, j.o0, j.n_tot, j.flip = 2, self.Cout, 1, 0, 0, 0
            out.append(j)
        return out

    def attach_lora(self, blocks: List[ConvLoraRef]) -> None:
        self.lora = blocks
        c = 0
        for b in blocks:
            if b.w_down.shape[1] != self.Cin or tuple(b.w_down.shape[2:]) != (3, 3) or b.w_up.shape[0] != self.Cout:
                raise _lib.HcpError("Conv2d LoRA block does not match its 3x3 host convolution")
            if b.rank > 64 or (c % 64) + b.rank > 64:
                c = (c + 63) // 64 * 64
            b.c0 = c
            c += b.rank
        self.r_tot, self.R = c, (c + 63) // 64 * 64
        dev = self.W.device
        z = lambda *shape: torch.zeros(shape, dtype=BF16, device=dev)   # noqa: E731
        self.dapp = any(b.branch is not None for b in blocks)
        self.Wdl = z(self.Cin, 3, 3, self.R)         # dgrad arrangement of the taps of W_down
        self.Bl = z(self.Cout, self.R)
        if self.dapp:
            # every block writes the rows of ITS branch's buffers only: T / U of a batch half come out with zeros in the columns of
            # the other branch, so the main convolution's LoRA segment, the dgrad through W_down and both gradient kernels stay unmasked
            self.Wt_br = {"n": z(self.R, 3, 3, self.Cin), "p": z(self.R, 3, 3, self.Cin)}
            self.BlT_br = {"n": z(self.R, self.Cout), "p": z(self.R, self.Cout)}
        else:
            self.Wt = z(self.R, 3, 3, self.Cin)      # forward weights of T = conv3x3(x, W_down)
            self.BlT = z(self.R, self.Cout)

    def jobs(self) -> List[_lib.LoraJob]:
        out = []
        for b in self.lora:                          # up-projection only (in_dim = 0): alpha*W_up -> Bl / BlT
            j = _lib.LoraJob()
            j.w_down, j.w_up, j.alpha = b.w_up.data_ptr(), b.w_up.data_ptr(), b.alpha
            j.rank, j.in_dim, j.out_dim = b.rank, 0, self.Cout
            j.c0, j.o0, j.out_tot, j.ld_r = b.c0, 0, self.Cout, self.R
            blt = self.BlT_br[b.branch] if self.dapp else self.BlT
            j.A, j.AT, j.Bl, j.BlT = self.Bl.data_ptr(), self.Bl.data_ptr(), self.Bl.data_ptr(), blt.data_ptr()
            out.append(j)
        return out

    def conv_jobs(self) -> List[_lib.LoraConvJob]:
        out = []
        for b in self.lora:
            j = _lib.LoraConvJob()
            j.w_down, j.rank, j.cin, j.c0, j.ld_r = b.w_down.data_ptr(), b.rank, self.Cin, b.c0, self.R
            j.flip = 1 if self.stride == 1 else 0
            j.wt, j.wd = (self.Wt_br[b.branch] if self.dapp else self.Wt).data_ptr(), self.Wdl.data_ptr()
            out.append(j)
        return out

    def slabs(self):
        out = []
        for q in range(self.R // 64):
            lo, hi = 64 * q, 64 * q + 64
            pieces = []
            for b in self.lora:
                a, e = max(lo, b.c0), min(hi, b.c0 + b.rank)
                if a < e:
                    pieces.append((b, a - b.c0, e - a, a - lo))
            if pieces:
                out.append((q, pieces))
        return out


# ----------------------------------------------------------------------------------------------------------------------
# linear (+LoRA, + fused residual)
# ----------------------------------------------------------------------------------------------------------------------
def _skinny_rows(pack: LinearPack, a_list, b_key: str, M: int, batch: int, out: torch.Tensor, n_out: int) -> None:
    """out[M, R] = sum_s A_s . B_s^T for the LoRA down-projections (T = x . A^T, U = dY . (alpha B)).  Plain groups: one GEMM.
    DAPP groups: one GEMM per batch half against the row-masked operand of that half's branch, so T / U come out with zeros
    in the columns of the other branch and everything downstream (main GEMM segment, dX, gradient kernel) stays unmasked."""
    R = pack.R

    def b_list_for(t):
        rows = min(n_out, t.shape[0])      # rows beyond the operand read as zero (merged packs keep only the 8-padded rank rows)
        if b_key == "A":       # [R, K] against the (possibly multi-input) x: column offsets follow the k splits
            bl, off = [], 0
            for (_, _, k) in a_list:
                bl.append((t, pack.K, rows, off))
                off += k
            return bl
        return [(t, pack.N, rows, 0)]

    if not pack.dapp:
        gemm_raw(a_list, b_list_for(pack.A if b_key == "A" else pack.BlT), M, R, out, R)
        return
    if batch % 2:
        raise _lib.HcpError("DreamArtist++ (dapp) layers need an even batch: [negative half | positive half]")
    Mh = M // 2
    for half, br in ((0, "n"), (1, "p")):
        t = (pack.A_br if b_key == "A" else pack.BlT_br)[br]
        rows = [(_RowView(a, half * Mh * lda), lda, k) for (a, lda, k) in a_list]
        gemm_raw(rows, b_list_for(t), Mh, R, _RowView(out, half * Mh * R), R)


class _RowView:
    """A row-offset alias of a bf16 matrix for gemm_raw (which only needs data_ptr())."""
    __slots__ = ("t", "off", "device")

    def __init__(self, t, elem_off: int):
        self.t, self.off, self.device = t, elem_off, t.device

    def data_ptr(self) -> int:
        return self.t.data_ptr() + 2 * self.off


class FusedLinearFn(torch.autograd.Function):
    """y = cat(xs, -1) . W^T + b (+ T . Bl^T, T = x . A^T)(+ residual).  Reference semantics:
    LoraPatchContainer.forward / LoraBlock.post_forward / LinearLayer.forward (hcpdiff/models/lora_base_patch.py:21-35,
    68-74, lora_layers_patch.py:44-57) and DAPPPatchContainer.forward (lora_layers_patch.py:102-133) without materialising
    W + alpha*W_up@W_down."""

    @staticmethod
    def forward(ctx, pack: LinearPack, residual: Optional[torch.Tensor], n_x: int, *tensors):
        xs = [_chk(t, "linear input") for t in tensors[:n_x]]
        ctx.n_extra = len(tensors) - n_x      # LoRA parameters: autograd inputs so the node exists even when x has no grad
        M = xs[0].numel() // xs[0].shape[-1]
        ks = [x.shape[-1] for x in xs]
        if ks != pack.k_splits:
            raise _lib.HcpError(f"linear: input widths {ks} do not match the packed weight splits {pack.k_splits}")
        N = pack.N
        out = torch.empty((*xs[0].shape[:-1], N), dtype=BF16, device=xs[0].device)
        a_list = [(x, k, k) for x, k in zip(xs, ks)]
        b_list, off = [], 0
        for k in ks:
            b_list.append(pack.b_fwd(off))
            off += k
        T = None
        if pack.lora and not pack.merged:
            if len(a_list) + 1 > _lib.MAX_SEG:
                raise _lib.HcpError("LoRA on a linear with more than two concatenated inputs is not supported")
            T = torch.empty((M, pack.R), dtype=BF16, device=xs[0].device)
            _skinny_rows(pack, list(a_list), "A", M, xs[0].shape[0], T, pack.R)
            a_list.append((T, pack.R, pack.r_tot))
            b_list.append((pack.Bl, pack.R, N, 0))
        res = None
        if residual is not None:
            res = _chk(residual, "linear residual")
        if pack.ext_rp and any(ctx.needs_input_grad[3 + n_x:]):
            # the factor gradients will need T = x W_down^T: it rides this GEMM as ext_rp extra output columns
            T = torch.empty((M, pack.R), dtype=BF16, device=xs[0].device)
            gemm_raw(a_list, [(pack.W, pack.K, N + pack.ext_rp, 0)], M, N + pack.ext_rp, out, N, bias=pack.bias, residual=res, ldr=N,
                     out2=T, ldo2=pack.R, n_main=N)
        else:
            if pack.ext_rp:
                b_list = [(pack.W, pack.K, N, 0)]
            gemm_raw(a_list, b_list, M, N, out, N, bias=pack.bias, residual=res, ldr=N)
        ctx.pack, ctx.n_x, ctx.M, ctx.ks = pack, n_x, M, ks
        ctx.batch = xs[0].shape[0]
        ctx.has_res = residual is not None
        saved = list(xs) if (pack.lora or pack.train) else []
        if T is not None:
            saved.append(T)
        ctx.save_for_backward(*saved)
        ctx.x_shapes = [x.shape for x in xs]
        return out

    @staticmethod
    def _lora_grads(pack, xs, ks, T, U, dy, M, N, R):
        for q, pieces in pack.slabs():
            for p0 in range(0, len(pieces), 8):
                chunk = pieces[p0:p0 + 8]
                nb = len(chunk)
                up = (_lib.LoraGradBlock * nb)()
                for i, (b, j0, rows, cs) in enumerate(chunk):
                    gu = b.g_up if b.g_up is not None else _acc_grad(b.w_up)
                    up[i].n_lo, up[i].n_hi, up[i].c0, up[i].rank = b.o0, b.o0 + b.out_dim, cs, rows
                    up[i].scale, up[i].transpose_out, up[i].dst, up[i].dst_ld = b.alpha, 1, gu.data_ptr() + 4 * j0, b.rank
                koff = 0
                for xi, (x, k) in enumerate(zip(xs, ks)):
                    down = (_lib.LoraGradBlock * nb)()
                    for i, (b, j0, rows, cs) in enumerate(chunk):
                        gd = b.g_down if b.g_down is not None else _acc_grad(b.w_down)
                        down[i].n_lo, down[i].n_hi, down[i].c0, down[i].rank = 0, k, cs, rows
                        down[i].scale, down[i].transpose_out = 1.0, 0
                        down[i].dst, down[i].dst_ld = gd.data_ptr() + 4 * (j0 * pack.K + koff), pack.K
                    Uq, Tq = U.data_ptr() + 2 * 64 * q, T.data_ptr() + 2 * 64 * q
                    if xi == 0:
                        call("hcp_lora_grad_pair", Uq, x.data_ptr(), k, k, down, Tq, dy.data_ptr(), N, N, up, nb, M, R, stream_ptr())
                    else:
                        call("hcp_lora_grad", Uq, R, x.data_ptr(), k, M, 0, k, down, nb, stream_ptr())
                    koff += k

    @staticmethod
    def backward(ctx, dy):
        pack, M, ks = ctx.pack, ctx.M, ctx.ks
        dy = _chk(dy, "linear grad")
        N, R = pack.N, pack.R
        U = None
        if pack.train:
            # full fine-tune: dW[o, k] += sum_m dY[m, o] x[m, k] per trained host (wgmma TN GEMM), db[o] += colsum(dY)
            xs_t = ctx.saved_tensors[:len(ks)]
            for w, b, o0, n in pack.train:
                gw = _acc_grad(w)
                koff = 0
                for x, k in zip(xs_t, ks):
                    call("hcp_wgrad_bf16", dy.data_ptr() + 2 * o0, N, n, x.data_ptr(), k, k, M, 1.0, gw.data_ptr() + 4 * koff, pack.K, 1, stream_ptr())
                    koff += k
                if b is not None and b.requires_grad:
                    call("hcp_colsum_bf16", dy.data_ptr() + 2 * o0, N, M, n, 0, 1.0, _acc_grad(b).data_ptr(), n, stream_ptr())
                notify_grad(w, b)
        dx_done = None
        if pack.merged:
            # merged weights: dX is a plain GEMM against W_eff^T; T = x A^T and U = dY (alpha B) exist only for the factor gradients
            # dW_down = U^T x, dW_up = alpha dY^T T -- the whole LoRA backward of the layer is off the critical path.  With the rank
            # rows riding the weight operands (ext_rp) T came out of the forward GEMM and U comes out of the dX GEMM.
            saved = list(ctx.saved_tensors)
            T_saved = saved.pop() if (pack.ext_rp and len(saved) > len(ks)) else None
            xs = saved
            Um = None
            if T_saved is not None and ctx.needs_input_grad[3]:
                dx_done = torch.empty(ctx.x_shapes[0], dtype=BF16, device=dy.device)
                Um = torch.empty((M, R), dtype=BF16, device=dy.device)
                gemm_raw([(dy, N, N)], [(pack.WT, N, pack.K + pack.ext_rp, 0)], M, pack.K + pack.ext_rp, dx_done, pack.K,
                         out2=Um, ldo2=R, n_main=pack.K)

            def lora_side(Tm, Um):
                if Tm is None:
                    Tm = torch.empty((M, R), dtype=BF16, device=dy.device)
                    _skinny_rows(pack, [(x, k, k) for x, k in zip(xs, ks)], "A", M, ctx.batch, Tm, R)
                if Um is None:
                    Um = torch.empty((M, R), dtype=BF16, device=dy.device)
                    _skinny_rows(pack, [(dy, N, N)], "BlT", M, ctx.batch, Um, R)
                FusedLinearFn._lora_grads(pack, xs, ks, Tm, Um, dy, M, N, R)
                return Tm, Um

            if side_enabled():
                side = fork_side(dy, T_saved, Um, *xs)
                with torch.cuda.stream(side):
                    tu = lora_side(T_saved, Um)
                _Side.keep.extend(tu)
            else:
                lora_side(T_saved, Um)
        elif pack.lora:
            *xs, T = ctx.saved_tensors
            U = torch.empty((M, R), dtype=BF16, device=dy.device)
            _skinny_rows(pack, [(dy, N, N)], "BlT", M, ctx.batch, U, R)
            # dW_down = U^T x ;  dW_up = alpha * dY^T T   (tensor-core TN GEMMs, one 64-column slab of U / T per launch).
            # Nothing downstream of this node reads them: with the side stream on they run next to the dX GEMM of the main chain.
            if side_enabled():
                with torch.cuda.stream(fork_side(U, T, dy, *xs)):
                    FusedLinearFn._lora_grads(pack, xs, ks, T, U, dy, M, N, R)
            else:
                FusedLinearFn._lora_grads(pack, xs, ks, T, U, dy, M, N, R)
        grads = []
        off = 0
        for i, k in enumerate(ks):
            if dx_done is not None:
                grads.append(dx_done)
            elif ctx.needs_input_grad[3 + i]:
                dx = torch.empty(ctx.x_shapes[i], dtype=BF16, device=dy.device)
                a_list = [(dy, N, N)]
                b_list = [pack.b_dgrad(off, k)]
                if U is not None:
                    a_list.append((U, R, pack.r_tot))
                    b_list.append((pack.AT, R, k, off * R))
                gemm_raw(a_list, b_list, M, k, dx, k)
                grads.append(dx)
            else:
                grads.append(None)
            off += k
        dres = dy if (ctx.has_res and ctx.needs_input_grad[1]) else None
        return (None, dres, None, *grads, *([None] * ctx.n_extra))


def _acc_grad(p: torch.Tensor) -> torch.Tensor:
    """fp32 .grad of a LoRA parameter, created zeroed on first use; the kernels accumulate into it directly."""
    if p.grad is None:
        p.grad = torch.zeros_like(p, dtype=torch.float32)
    return p.grad


def fused_linear(pack: LinearPack, xs: Sequence[torch.Tensor], residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    # The LoRA parameters are passed as autograd inputs so the node is recorded even when x carries no gradient (cross-attention
    # k/v on the text embedding); their gradients are accumulated in place by the kernels (fp32 .grad / flat grad buffer).
    extra = []
    for b in pack.lora:
        extra += [b.w_down, b.w_up]
    for w, _, _, _ in pack.train:
        extra.append(w)
    return FusedLinearFn.apply(pack, residual, len(xs), *xs, *extra)


# ----------------------------------------------------------------------------------------------------------------------
# 3x3 convolution
# ----------------------------------------------------------------------------------------------------------------------
class Conv3x3Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pack: ConvPack, geom: Tuple[int, int, int], rowbias: Optional[torch.Tensor], residual: Optional[torch.Tensor],
                x: torch.Tensor, *lora_params):
        B, H, W = geom
        x = _chk(x, "conv input")
        s = pack.stride
        Ho, Wo = H // s, W // s
        out = torch.empty((B, Ho * Wo, pack.Cout), dtype=BF16, device=x.device)
        res = None if residual is None else _chk(residual, "conv residual")
        rb_ld = 0
        if rowbias is not None:
            if rowbias.dtype != torch.float32 or rowbias.stride(-1) != 1:
                raise _lib.HcpError("conv rowbias must be fp32 with unit inner stride")
            rb_ld = rowbias.stride(0)
        T, lora = None, None
        if pack.lora:
            T = torch.empty((B, Ho * Wo, pack.R), dtype=BF16, device=x.device)
            if not pack.dapp:
                conv3x3_raw(x, pack.Wt, B, H, W, pack.Cin, pack.R, s, 0, T)               # T = conv3x3(x, W_down)
            else:                                    # DreamArtist++: one launch per batch half against that half's branch rows
                if B % 2:
                    raise _lib.HcpError("DreamArtist++ (dapp) layers need an even batch: [negative half | positive half]")
                Bh = B // 2
                for half, br in ((0, "n"), (1, "p")):
                    conv3x3_raw(_RowView(x, half * Bh * H * W * pack.Cin), pack.Wt_br[br], Bh, H, W, pack.Cin, pack.R, s, 0,
                                _RowView(T, half * Bh * Ho * Wo * pack.R))
            lora = (T, pack.Bl, pack.r_tot, pack.R)
        conv3x3_raw(x, pack.W, B, H, W, pack.Cin, pack.Cout, s, 0, out, bias=pack.bias, rowbias=rowbias, residual=res, rowbias_ld=rb_ld,
                    lora=lora, w_tiled=pack.tiled)
        ctx.pack, ctx.geom = pack, geom
        ctx.has_res = residual is not None
        ctx.n_extra = len(lora_params)
        if pack.lora:
            ctx.save_for_backward(x, T)
        elif pack.train is not None:
            ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, dy):
        pack = ctx.pack
        B, H, W = ctx.geom
        dy = _chk(dy, "conv grad")
        s = pack.stride
        M = B * (H // s) * (W // s)
        U = None
        if pack.train is not None:
            # full fine-tune: dW [Cout, Cin, 3, 3] += dY^T x_shifted (nine TN GEMMs over the shifted NHWC boxes), db += colsum(dY)
            w, b = pack.train
            call("hcp_wgrad_conv3x3_bf16", dy.data_ptr(), pack.Cout, ctx.saved_tensors[0].data_ptr(), B, H, W, pack.Cin, s, 1.0,
                 _acc_grad(w).data_ptr(), stream_ptr())
            if b is not None and b.requires_grad:
                call("hcp_colsum_bf16", dy.data_ptr(), pack.Cout, M, pack.Cout, 0, 1.0, _acc_grad(b).data_ptr(), pack.Cout, stream_ptr())
            notify_grad(w, b)
        d_rowbias = None
        if ctx.needs_input_grad[2]:
            # the per-image row bias is the time-embedding projection: d temb[b, c] = sum over the image's pixels of dY
            d_rowbias = torch.zeros((B, pack.Cout), dtype=torch.float32, device=dy.device)
            call("hcp_colsum_bf16", dy.data_ptr(), pack.Cout, M, pack.Cout, M // B, 1.0, d_rowbias.data_ptr(), pack.Cout, stream_ptr())
        if pack.lora:
            x, T = ctx.saved_tensors
            R, N = pack.R, pack.Cout
            U = torch.empty((M, R), dtype=BF16, device=dy.device)
            if not pack.dapp:
                gemm_raw([(dy, N, N)], [(pack.BlT, N, R, 0)], M, R, U, R)                   # U = dY . (alpha W_up)
            else:
                Mh = M // 2
                for half, br in ((0, "n"), (1, "p")):
                    gemm_raw([(_RowView(dy, half * Mh * N), N, N)], [(pack.BlT_br[br], N, R, 0)], Mh, R, _RowView(U, half * Mh * R), R)
            for q, pieces in pack.slabs():
                for p0 in range(0, len(pieces), 8):
                    chunk = pieces[p0:p0 + 8]
                    nb = len(chunk)
                    up = (_lib.LoraGradBlock * nb)()
                    down = (_lib.LoraGradBlock * nb)()
                    for i, (b, j0, rows, cs) in enumerate(chunk):
                        gu, gd = _acc_grad(b.w_up), _acc_grad(b.w_down)
                        up[i].n_lo, up[i].n_hi, up[i].c0, up[i].rank = 0, N, cs, rows
                        up[i].scale, up[i].transpose_out, up[i].dst, up[i].dst_ld = b.alpha, 1, gu.data_ptr() + 4 * j0, b.rank
                        down[i].c0, down[i].rank, down[i].scale = cs, rows, 1.0
                        down[i].dst = gd.data_ptr() + 4 * j0 * pack.Cin * 9
                    # dW_up = alpha dY^T T ;  dW_down[., ., kh, kw] = U^T x_shifted(kh, kw)
                    call("hcp_lora_grad", T.data_ptr() + 2 * 64 * q, R, dy.data_ptr(), N, M, 0, N, up, nb, stream_ptr())
                    call("hcp_lora_grad_conv3x3", U.data_ptr() + 2 * 64 * q, R, x.data_ptr(), B, H, W, pack.Cin, s, down, nb, stream_ptr())
        dx = None
        if ctx.needs_input_grad[4]:
            dx = torch.empty((B, H * W, pack.Cin), dtype=BF16, device=dy.device)
            if s == 1:
                conv3x3_raw(dy, pack.Wd, B, H, W, pack.Cout, pack.Cin, 1, 0, dx, w_tiled=pack.tiled)
                if U is not None:                                                           # + dgrad through W_down
                    conv3x3_raw(U, pack.Wdl, B, H, W, pack.R, pack.Cin, 1, 0, dx, residual=dx)
            else:
                conv3x3_raw(dy, pack.Wd, B, H // 2, W // 2, pack.Cout, pack.Cin, 2, 1, dx, w_tiled=pack.tiled)
                if U is not None:
                    conv3x3_raw(U, pack.Wdl, B, H // 2, W // 2, pack.R, pack.Cin, 2, 1, dx, residual=dx)
        dres = dy if (ctx.has_res and ctx.needs_input_grad[3]) else None
        return (None, None, d_rowbias, dres, dx, *([None] * ctx.n_extra))


def conv3x3(pack: ConvPack, x: torch.Tensor, geom, rowbias=None, residual=None) -> torch.Tensor:
    extra = []
    for b in pack.lora:          # autograd inputs so the node exists even when x carries no gradient
        extra += [b.w_down, b.w_up]
    if pack.train is not None:
        extra.append(pack.train[0])
    return Conv3x3Fn.apply(pack, geom, rowbias, residual, x, *extra)


# ----------------------------------------------------------------------------------------------------------------------
# normalisation
# ----------------------------------------------------------------------------------------------------------------------
class GroupNormFn(torch.autograd.Function):
    """(y, alias(x1)[, alias(x2)]) = GN(cat(x1, x2)) [+SiLU]; the aliases carry the residual-branch gradients back so the
    fan-in add happens inside the GroupNorm backward kernel."""

    @staticmethod
    def forward(ctx, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool, x1: torch.Tensor,
                x2: Optional[torch.Tensor]):
        x1 = _chk(x1, "groupnorm input")
        B, HW, C1 = x1.shape
        C2 = 0
        if x2 is not None:
            x2 = _chk(x2, "groupnorm input 2")
            C2 = x2.shape[-1]
        y = torch.empty((B, HW, C1 + C2), dtype=BF16, device=x1.device)
        stats = torch.empty((B, groups, 2), dtype=torch.float32, device=x1.device)
        wsb = _lib.lib().hcp_groupnorm_workspace_bytes(B, HW, groups)
        ws = torch.empty((max(wsb, 4) // 4,), dtype=torch.float32, device=x1.device)
        a = GroupNormArgs()
        a.x1, a.x2 = x1.data_ptr(), ptr(x2)
        a.B, a.HW, a.C1, a.C2, a.G = B, HW, C1, C2, groups
        a.gamma, a.beta, a.eps, a.silu = gamma.data_ptr(), beta.data_ptr(), eps, int(silu)
        a.stats, a.workspace, a.workspace_bytes = stats.data_ptr(), ws.data_ptr(), wsb
        a.y = y.data_ptr()
        call("hcp_groupnorm_fwd_bf16", C.byref(a), stream_ptr())
        ctx.set_materialize_grads(False)      # an unused alias output must arrive as None in backward, not as a zero-filled tensor
        ctx.save_for_backward(x1, x2, stats, gamma, beta)
        ctx.cfg = (groups, eps, silu)
        if x2 is None:
            return y, x1
        return y, x1, x2

    @staticmethod
    def backward(ctx, dy, d1, d2=None):
        x1, x2, stats, gamma, beta = ctx.saved_tensors
        groups, eps, silu = ctx.cfg
        B, HW, C1 = x1.shape
        C2 = 0 if x2 is None else x2.shape[-1]
        need1 = ctx.needs_input_grad[5]
        need2 = x2 is not None and ctx.needs_input_grad[6]
        if not (need1 or need2 or gamma.requires_grad):
            return (None,) * 7
        if dy is None:
            return None, None, None, None, None, d1, d2
        dy = _chk(dy, "groupnorm grad")
        if gamma.requires_grad:       # full fine-tune: dgamma / dbeta accumulate straight into the parameters' fp32 gradients
            call("hcp_norm_affine_grad_bf16", x1.data_ptr(), ptr(x2), C1, C2, dy.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                 B * HW, HW, groups, int(silu), _acc_grad(gamma).data_ptr(), _acc_grad(beta).data_ptr(), stream_ptr())
            notify_grad(gamma, beta)
        dx1 = torch.empty_like(x1)
        dx2 = None if x2 is None else torch.empty_like(x2)
        wsb = _lib.lib().hcp_groupnorm_workspace_bytes(B, HW, groups)
        ws = torch.empty((max(wsb, 4) // 4,), dtype=torch.float32, device=x1.device)
        a = GroupNormArgs()
        a.x1, a.x2 = x1.data_ptr(), ptr(x2)
        a.B, a.HW, a.C1, a.C2, a.G = B, HW, C1, C2, groups
        a.gamma, a.beta, a.eps, a.silu = gamma.data_ptr(), beta.data_ptr(), eps, int(silu)
        a.stats, a.workspace, a.workspace_bytes = stats.data_ptr(), ws.data_ptr(), wsb
        a.dy = dy.data_ptr()
        a.add1 = None if d1 is None else _chk(d1, "groupnorm alias grad").data_ptr()
        a.add2 = None if d2 is None else _chk(d2, "groupnorm alias grad 2").data_ptr()
        a.dx1, a.dx2 = dx1.data_ptr(), ptr(dx2)
        call("hcp_groupnorm_bwd_bf16", C.byref(a), stream_ptr())
        return None, None, None, None, None, dx1, dx2


def group_norm(gamma, beta, groups, eps, silu, x1, x2=None):
    return GroupNormFn.apply(gamma, beta, groups, eps, silu, x1, x2)


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gamma: torch.Tensor, beta: torch.Tensor, eps: float, x: torch.Tensor):
        x = _chk(x, "layernorm input")
        C_ = x.shape[-1]
        M = x.numel() // C_
        y = torch.empty_like(x)
        stats = torch.empty((M, 2), dtype=torch.float32, device=x.device)
        call("hcp_layernorm_fwd_bf16", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, M, C_, stats.data_ptr(), y.data_ptr(),
             stream_ptr())
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, stats, gamma, beta)
        return y, x

    @staticmethod
    def backward(ctx, dy, dalias):
        x, stats, gamma, beta = ctx.saved_tensors
        if not ctx.needs_input_grad[3] and not gamma.requires_grad:
            return None, None, None, None
        if dy is None:
            return None, None, None, dalias
        dy = _chk(dy, "layernorm grad")
        C_ = x.shape[-1]
        M = x.numel() // C_
        if gamma.requires_grad:
            call("hcp_norm_affine_grad_bf16", x.data_ptr(), None, C_, 0, dy.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                 M, 0, 0, 0, _acc_grad(gamma).data_ptr(), _acc_grad(beta).data_ptr(), stream_ptr())
            notify_grad(gamma, beta)
        dx = torch.empty_like(x)
        add = None if dalias is None else _chk(dalias, "layernorm alias grad")
        call("hcp_layernorm_bwd_bf16", x.data_ptr(), dy.data_ptr(), ptr(add), gamma.data_ptr(), stats.data_ptr(), M, C_, dx.data_ptr(),
             stream_ptr())
        return None, None, None, dx


def layer_norm(gamma, beta, eps, x):
    return LayerNormFn.apply(gamma, beta, eps, x)


# ----------------------------------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------------------------------
class AttentionFn(torch.autograd.Function):
    """softmax(q k^T * scale + bias) v over heads laid out as column blocks.
    q_src [B,Lq,ldq] holds q at column q_off; kv_src [B,Lkv,ldkv] holds k at k_off and v at v_off (q_src may be kv_src:
    the fused QKV projection output)."""

    @staticmethod
    def forward(ctx, heads: int, C_: int, offs: Tuple[int, int, int], kv_bias: Optional[torch.Tensor], q_src: torch.Tensor,
                kv_src: Optional[torch.Tensor]):
        q_src = _chk(q_src, "attention q")
        same = kv_src is None
        kvt = q_src if same else _chk(kv_src, "attention kv")
        B, Lq, ldq = q_src.shape
        _, Lkv, ldkv = kvt.shape
        d = C_ // heads
        scale = 1.0 / math.sqrt(d)
        o = torch.empty((B, Lq, C_), dtype=BF16, device=q_src.device)
        lse = torch.empty((B, heads, Lq), dtype=torch.float32, device=q_src.device)
        a = AttnArgs()
        a.q, a.ldq = q_src.data_ptr() + 2 * offs[0], ldq
        a.k, a.ldk = kvt.data_ptr() + 2 * offs[1], ldkv
        a.v, a.ldv = kvt.data_ptr() + 2 * offs[2], ldkv
        a.B, a.H, a.Lq, a.Lkv, a.d = B, heads, Lq, Lkv, d
        a.scale = scale
        a.kv_bias = ptr(kv_bias)
        a.o, a.ldo, a.lse = o.data_ptr(), C_, lse.data_ptr()
        call("hcp_attn_fwd_bf16", C.byref(a), stream_ptr())
        ctx.save_for_backward(q_src, kvt, o, lse, kv_bias)
        ctx.cfg = (heads, C_, offs, same, scale)
        return o

    @staticmethod
    def backward(ctx, do):
        q_src, kvt, o, lse, kv_bias = ctx.saved_tensors
        heads, C_, offs, same, scale = ctx.cfg
        do = _chk(do, "attention grad")
        B, Lq, ldq = q_src.shape
        _, Lkv, ldkv = kvt.shape
        d = C_ // heads
        # gradients are written straight into buffers with the layout of the sources
        dq_src = torch.empty_like(q_src)
        dkv = dq_src if same else torch.empty_like(kvt)
        wsb = _lib.lib().hcp_attn_bwd_workspace_bytes(B, heads, Lq, Lkv, d)
        ws = torch.empty((wsb // 4,), dtype=torch.float32, device=do.device)
        a = AttnBwdArgs()
        a.q, a.ldq = q_src.data_ptr() + 2 * offs[0], ldq
        a.k, a.ldk = kvt.data_ptr() + 2 * offs[1], ldkv
        a.v, a.ldv = kvt.data_ptr() + 2 * offs[2], ldkv
        a.o, a.ldo, a.dout, a.lddo = o.data_ptr(), C_, do.data_ptr(), C_
        a.B, a.H, a.Lq, a.Lkv, a.d = B, heads, Lq, Lkv, d
        a.scale, a.kv_bias, a.lse = scale, ptr(kv_bias), lse.data_ptr()
        a.dq, a.lddq = dq_src.data_ptr() + 2 * offs[0], ldq
        a.dk, a.lddk = dkv.data_ptr() + 2 * offs[1], ldkv
        a.dv, a.lddv = dkv.data_ptr() + 2 * offs[2], ldkv
        a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
        call("hcp_attn_bwd_bf16", C.byref(a), stream_ptr())
        return None, None, None, None, dq_src, (None if same else dkv)


def attention(heads: int, C_: int, offs, q_src, kv_src=None, kv_bias=None):
    return AttentionFn.apply(heads, C_, tuple(offs), kv_bias, q_src, kv_src)


# ----------------------------------------------------------------------------------------------------------------------
# elementwise
# ----------------------------------------------------------------------------------------------------------------------
class GegluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u):
        u = _chk(u, "geglu input")
        F2 = u.shape[-1]
        F_ = F2 // 2
        M = u.numel() // F2
        h = torch.empty((*u.shape[:-1], F_), dtype=BF16, device=u.device)
        call("hcp_geglu_fwd_bf16", u.data_ptr(), M, F_, h.data_ptr(), stream_ptr())
        ctx.save_for_backward(u)
        return h

    @staticmethod
    def backward(ctx, dh):
        (u,) = ctx.saved_tensors
        dh = _chk(dh, "geglu grad")
        F2 = u.shape[-1]
        M = u.numel() // F2
        du = torch.empty_like(u)
        call("hcp_geglu_bwd_bf16", u.data_ptr(), dh.data_ptr(), M, F2 // 2, du.data_ptr(), stream_ptr())
        return du


class Upsample2xFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, geom, x):
        B, H, W = geom
        x = _chk(x, "upsample input")
        C_ = x.shape[-1]
        y = torch.empty((B, 4 * H * W, C_), dtype=BF16, device=x.device)
        call("hcp_upsample2x_fwd_bf16", x.data_ptr(), B, H, W, C_, y.data_ptr(), stream_ptr())
        ctx.geom = geom
        return y

    @staticmethod
    def backward(ctx, dy):
        B, H, W = ctx.geom
        dy = _chk(dy, "upsample grad")
        C_ = dy.shape[-1]
        dx = torch.empty((B, H * W, C_), dtype=BF16, device=dy.device)
        call("hcp_upsample2x_bwd_bf16", dy.data_ptr(), B, H, W, C_, dx.data_ptr(), stream_ptr())
        return None, dx


class Fork2Fn(torch.autograd.Function):
    """Two aliases of one tensor whose gradients are summed by our own kernel (skip connections)."""

    @staticmethod
    def forward(ctx, x):
        return x, x

    @staticmethod
    def backward(ctx, da, db):
        if da is None:
            return db
        if db is None:
            return da
        da, db = _chk(da, "fork grad"), _chk(db, "fork grad")
        out = torch.empty_like(da)
        call("hcp_add_bf16", da.data_ptr(), db.data_ptr(), da.numel(), out.data_ptr(), stream_ptr())
        return out


class ConvOutFn(torch.autograd.Function):
    """bf16 NHWC [B,HW,Cin] -> fp32 NCHW [B,4,H,W] 3x3 convolution at the module boundary.  `train` = (weight, bias) Parameters of the
    nn.Conv2d when conv_out is trained (full fine-tune): their gradients are accumulated in place."""

    @staticmethod
    def forward(ctx, w: torch.Tensor, bias: Optional[torch.Tensor], geom, train, x):
        B, H, W = geom
        x = _chk(x, "conv_out input")
        Cin, Cout = x.shape[-1], w.shape[2]            # w: tap-major [3,3,Cout,Cin]
        y = torch.empty((B, Cout, H, W), dtype=torch.float32, device=x.device)
        call("hcp_conv_out_f32", x.data_ptr(), w.data_ptr(), ptr(bias), B, H, W, Cin, Cout, y.data_ptr(), stream_ptr())
        ctx.w, ctx.geom, ctx.Cin, ctx.train = w, geom, Cin, train
        if train is not None:
            ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, H, W = ctx.geom
        dy = dy.float().contiguous()
        Cout = ctx.w.shape[2]
        if ctx.train is not None:
            (x,) = ctx.saved_tensors
            wp, bp = ctx.train
            call("hcp_conv_out_wgrad_f32", dy.data_ptr(), x.data_ptr(), B, H, W, ctx.Cin, Cout, _acc_grad(wp).data_ptr(),
                 None if bp is None else _acc_grad(bp).data_ptr(), stream_ptr())
            notify_grad(wp, bp)
        dx = torch.empty((B, H * W, ctx.Cin), dtype=BF16, device=dy.device)
        call("hcp_conv_out_dgrad_f32", dy.data_ptr(), ctx.w.data_ptr(), B, H, W, ctx.Cin, Cout, dx.data_ptr(), stream_ptr())
        return None, None, None, None, dx


class ConvInFn(torch.autograd.Function):
    """fp32 NCHW latent -> bf16 NHWC [B, H*W, Cout].  The latent is data (no input gradient); with `train` = (weight, bias) Parameters
    the backward accumulates the nn.Conv2d-layout weight / bias gradients (full fine-tune)."""

    @staticmethod
    def forward(ctx, w: torch.Tensor, bias: Optional[torch.Tensor], train, wparam, x):
        B, Cin, H, W = x.shape
        Cout = w.shape[3]                              # w: tap-major [Cin,3,3,Cout]
        y = torch.empty((B, H * W, Cout), dtype=BF16, device=x.device)
        call("hcp_conv_in_f32", x.data_ptr(), w.data_ptr(), ptr(bias), B, Cin, H, W, Cout, y.data_ptr(), stream_ptr())
        ctx.train, ctx.dims = train, (B, Cin, H, W, Cout)
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dh):
        (x,) = ctx.saved_tensors
        B, Cin, H, W, Cout = ctx.dims
        dh = _chk(dh, "conv_in grad")
        wp, bp = ctx.train
        call("hcp_conv_in_wgrad_f32", dh.data_ptr(), x.data_ptr(), B, Cin, H, W, Cout, _acc_grad(wp).data_ptr(),
             None if bp is None else _acc_grad(bp).data_ptr(), stream_ptr())
        notify_grad(wp, bp)
        return None, None, None, None, None


def conv_in(x_nchw: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], train=None) -> torch.Tensor:
    """fp32 NCHW latent -> bf16 NHWC [B, H*W, Cout] (no input gradient: the latent is data)."""
    x = x_nchw.float().contiguous()
    if train is not None:
        return ConvInFn.apply(w, bias, train, train[0], x)       # the weight Parameter is an autograd input so that the node exists
    B, Cin, H, W = x.shape
    Cout = w.shape[3]                                  # w: tap-major [Cin,3,3,Cout]
    y = torch.empty((B, H * W, Cout), dtype=BF16, device=x.device)
    call("hcp_conv_in_f32", x.data_ptr(), w.data_ptr(), ptr(bias), B, Cin, H, W, Cout, y.data_ptr(), stream_ptr())
    return y


class SmallLinearFn(torch.autograd.Function):
    """y = act(x W^T + b) on fp32 rows (M = batch): the time-embedding MLP and the 22 time_emb_proj layers when they are trained or
    carry a gradient (full fine-tune).  `w_bf16` is the operand the forward kernel reads (repacked from the fp32 master every step);
    `train` = [(weight Parameter, bias Parameter or None, first row, rows)] -- one entry per nn.Linear stacked into `w_bf16`."""

    @staticmethod
    def forward(ctx, w_bf16: torch.Tensor, bias: Optional[torch.Tensor], silu: bool, train, anchor, x: torch.Tensor):
        x = x.float().contiguous()
        N, K = w_bf16.shape
        M = x.shape[0]
        z = torch.empty((M, N), dtype=torch.float32, device=x.device)
        call("hcp_skinny_linear", x.data_ptr(), w_bf16.data_ptr(), ptr(bias), M, K, N, 0, 0, z.data_ptr(), stream_ptr())
        y = z
        if silu:
            y = torch.empty_like(z)
            call("hcp_silu_f32", z.data_ptr(), None, z.numel(), y.data_ptr(), stream_ptr())
        ctx.save_for_backward(x, z, w_bf16)
        ctx.silu, ctx.train = silu, train
        return y

    @staticmethod
    def backward(ctx, dy):
        x, z, w_bf16 = ctx.saved_tensors
        N, K = w_bf16.shape
        M = x.shape[0]
        dy = dy.float().contiguous()
        if ctx.silu:
            dz = torch.empty_like(dy)
            call("hcp_silu_f32", z.data_ptr(), dy.data_ptr(), z.numel(), dz.data_ptr(), stream_ptr())
        else:
            dz = dy
        dx = torch.empty_like(x) if ctx.needs_input_grad[5] else None
        call("hcp_small_linear_bwd_f32", dz.data_ptr(), N, None, w_bf16.data_ptr(), M, N, K, ptr(dx), None, None, stream_ptr()) if dx is not None else None
        for wp, bp, o0, n in ctx.train or []:
            call("hcp_small_linear_bwd_f32", dz.data_ptr() + 4 * o0, N, x.data_ptr(), None, M, n, K, None, _acc_grad(wp).data_ptr(),
                 None if bp is None else _acc_grad(bp).data_ptr(), stream_ptr())
            notify_grad(wp, bp)
        return None, None, None, None, None, dx


def small_linear(x, w_bf16, bias, silu, train=None):
    anchor = train[0][0] if train else None
    return SmallLinearFn.apply(w_bf16, bias, silu, train, anchor, x)


def skinny_linear(x: torch.Tensor, w_bf16: torch.Tensor, bias: Optional[torch.Tensor], in_mode: int, out_silu: bool) -> torch.Tensor:
    """fp32 [M<=16, K] (or timesteps [M] when in_mode == 2) -> fp32 [M, N]."""
    N, K = w_bf16.shape
    M = x.shape[0]
    y = torch.empty((M, N), dtype=torch.float32, device=w_bf16.device)
    call("hcp_skinny_linear", x.data_ptr(), w_bf16.data_ptr(), ptr(bias), M, K, N, in_mode, int(out_silu), y.data_ptr(), stream_ptr())
    return y


def sinusoid(x: torch.Tensor, dim: int, per_row: int, out: torch.Tensor, col0: int) -> None:
    """out[m // per_row, col0 + (m % per_row) * dim + j] = sinusoidal embedding (cos | sin) of x[m]; out fp32 2-D, x fp32 [M]."""
    call("hcp_sinusoid_f32", x.data_ptr(), x.numel(), dim, per_row, out.data_ptr() + 4 * col0, out.stride(0), stream_ptr())


def cast_bf16(x: torch.Tensor) -> torch.Tensor:
    x = x.float().contiguous()
    y = torch.empty(x.shape, dtype=BF16, device=x.device)
    call("hcp_cast_f32_to_bf16", x.data_ptr(), x.numel(), y.data_ptr(), stream_ptr())
    return y
