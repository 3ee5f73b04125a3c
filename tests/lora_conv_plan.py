"""Host-side planners of the Conv2d LoRA (LoCon) path, restated in Python, and the case lists of tests/test_gpu_lora_conv_edges.py.
tests/test_lora_conv_plan.py checks on the CPU that the cases reach every branch; the GPU tests use the same functions to name the
path a case takes and the tiles its errors are measured over.

  tile_n        pick_bn (gemm.cu): column-tile width BN of the GEMM / convolution kernel
  split_plan    plan_splits + run_gemm + hcp_splitk_workspace_bytes (gemm.cu) for a convolution with total_k = 9 Cin + R: the number
                of K-splits, k-blocks per split, and the split that holds the LoRA K-segment's k-blocks
  conv_box      plan_conv_box (host_util.cu): the 128-pixel box (bw x bh pixels x bnimg images) of every 3x3 convolution kernel:
                hcp_conv3x3_bf16 (mode 0), hcp_wgrad_conv3x3_bf16 and hcp_lora_grad_conv3x3
  lora_grad_plan  hcp_lora_grad_conv3x3's grid: 128-column chunks of Cin and the row split of the 128-row tiles
  lora_layout   lora_columns (ops.py, both packs' attach_lora): the first rank column c0 of each block, r_tot and the 64-padded R
  slabs         lora_slabs (ops.py): the pieces of each 64-column slab the gradient kernel reduces, 8 per launch
"""
H100_SMS = 132          # H100 SXM; the GPU tests re-plan with the live SM count
BLOCK_K = 64


def tile_n(N):
    """Column-tile width BN the GEMM / convolution kernel picks for N output columns (pick_bn in gemm.cu): the error blocks."""
    if N <= 64 or (N % 64 == 0 and N < 256 and N % 128):
        return 32 if N <= 32 else 64
    return min((128, 160, 176), key=lambda c: ((N + c - 1) // c * c, -c))


def plan_splits(ctas, total_kb, N, sms=H100_SMS):
    if total_kb < 8 or N <= 64:
        return 1, "short"
    if ctas >= sms // 3:
        return (2, "halves") if ctas <= sms // 2 and total_kb >= 40 else (1, "busy")
    s = min(sms // ctas, total_kb // 4, 16)
    return (1, "wave") if s < 2 else (s, "wave")


def conv_box(B, H, W, stride):
    """128-pixel box of a mode-0 convolution, and of both weight-gradient kernels, on an H x W input (plan_conv_box in host_util.cu)."""
    oH, oW = H // stride, W // stride
    if oW >= 128:
        assert oW % 128 == 0
        bw, bh, bnimg = 128, 1, 1
    else:
        assert 128 % oW == 0
        bw, bh = oW, 128 // oW
        if bh <= oH:
            assert oH % bh == 0
            bnimg = 1
        else:
            bh = oH
            assert 128 % (bw * bh) == 0
            bnimg = 128 // (bw * bh)
    tiles_w, tiles_h = oW // bw, oH // bh
    m_tiles = B * tiles_w * tiles_h if bnimg == 1 else -(-B // bnimg)
    return {"bw": bw, "bh": bh, "bnimg": bnimg, "tiles_w": tiles_w, "tiles_h": tiles_h, "m_tiles": m_tiles}


def split_plan(B, H, W, Cin, Cout, stride, R, r_tot, sms=H100_SMS):
    """K-splits of the forward convolution with its LoRA segment (R: the row pitch the workspace is sized from, r_tot: the rank
    columns read).  lora_split: the 0-based split that holds the LoRA k-blocks; lora_alone: that split holds no convolution k-block."""
    box = conv_box(B, H, W, stride)
    ctas = box["m_tiles"] * -(-Cout // tile_n(Cout))
    conv_kb, lora_kb = 9 * Cin // BLOCK_K, -(-r_tot // BLOCK_K)
    assert lora_kb == -(-R // BLOCK_K)          # the workspace is sized from R, the launch plans from r_tot: the same k-block count
    total_kb = conv_kb + lora_kb
    splits, branch = plan_splits(ctas, total_kb, Cout, sms)
    per = total_kb
    if splits > 1:
        per = -(-total_kb // splits)
        splits = -(-total_kb // per)
    return {"ctas": ctas, "total_kb": total_kb, "splits": splits, "branch": branch, "kb_per_split": per,
            "lora_split": conv_kb // per, "lora_alone": splits > 1 and conv_kb % per == 0}


def lora_grad_plan(B, H, W, Cin, stride, sms=H100_SMS):
    M = B * (H // stride) * (W // stride)
    col_chunks = -(-Cin // 128)
    total = -(-M // 128)
    splits = min(total, max(1, sms // col_chunks))
    per = -(-total // splits)
    return {"col_chunks": col_chunks, "part_chunk": Cin % 128 != 0, "splits": -(-total // per), "tiles_per_cta": per}


def lora_layout(ranks):
    """-> ([c0 of each block], r_tot, R): a block that would cross a 64-column boundary (or is wider than 64) starts a new slab."""
    c, c0s = 0, []
    for r in ranks:
        if r > 64 or c % 64 + r > 64:
            c = (c + 63) // 64 * 64
        c0s.append(c)
        c += r
    return c0s, c, (c + 63) // 64 * 64


def slabs(ranks):
    """[(slab, [(block index, first rank row j0, rows, first column inside the slab)])], as lora_slabs in ops.py."""
    c0s, _, R = lora_layout(ranks)
    out = []
    for q in range(R // 64):
        lo, hi = 64 * q, 64 * q + 64
        pieces = [(i, max(lo, c0) - c0, min(hi, c0 + r) - max(lo, c0), max(lo, c0) - lo)
                  for i, (c0, r) in enumerate(zip(c0s, ranks)) if max(lo, c0) < min(hi, c0 + r)]
        if pieces:
            out.append((q, pieces))
    return out


def klast(r):
    """16-wide k-steps in the last k-block of a LoRA segment of r rank columns (conv_lora_segment)."""
    return (r - (-(-r // BLOCK_K) - 1) * BLOCK_K + 15) // 16


def dapp_straddles(B, H, W, stride):
    """A 128-row tile of the main convolution holds rows of both batch halves (DreamArtist++: [negative | positive])."""
    return (B // 2) * (H // stride) * (W // stride) % 128 != 0


# ---------------------------------------------------------------------------------------------------------------------------------
# case lists: (B, H, W, Cin, Cout, stride, ranks)
# ---------------------------------------------------------------------------------------------------------------------------------
CASES = [
    (1, 128, 128, 320, 320, 1, (16,)),            # SDXL LoCon top level: one-row 128-pixel boxes, three column chunks (part-filled)
    (1, 128, 128, 320, 320, 2, (16,)),            # its downsampler: 64 x 2 boxes, the 5-D phase view
    (1, 2, 256, 64, 64, 1, (20,)),                # two boxes per row; rank 20: a partial last k-step
    (2, 8, 8, 1280, 1280, 1, (16,)),              # 8x8 level: 16 K-splits, the last one holds only the LoRA k-block
    (3, 2, 2, 64, 64, 1, (4, 8)),                 # 32 images a tile, the last tile part-filled; r_tot 12
    (3, 4, 4, 64, 128, 2, (80,)),                 # stride 2 to 2x2; rank 80 over two slabs (R 128)
    (2, 16, 16, 256, 64, 1, (40, 40, 40)),        # slab-alignment gaps, R 192; two column chunks
    (2, 16, 16, 64, 64, 1, (4,) * 9),             # nine blocks in one slab: two launches of each gradient kernel
    (2, 16, 16, 320, 640, 1, (64,)),              # part-filled column chunk; 8 K-splits, the LoRA k-block shares the last one
    (2, 32, 32, 64, 64, 2, (4,)),                 # stride 2 with Cin 64: the second half-box of the chunk reads phase-1 data
    (2, 64, 64, 320, 128, 1, (36,)),              # two K halves (64 output tiles), the LoRA k-block in the second
]
# dW_up (hcp_lora_grad, transpose_out = 1): (M, Cout, ranks) -- 3 / 5 column chunks of dY, the last part-filled
UP_CASES = [(16384, 320, (16,)), (512, 640, (64,)), (300, 320, (4,) * 9), (48, 640, (40, 40, 40))]
# DreamArtist++ on a 3x3 host: (B, H, W, Cin, Cout, stride, ranks of the 'n' blocks, ranks of the 'p' blocks)
DAPP_CASES = [
    (6, 4, 4, 64, 64, 1, (4,), (8,)),             # 8 images a tile: the only tile holds both halves
    (4, 16, 16, 64, 128, 2, (8,), (4, 20)),       # halves of one tile each
    (2, 16, 16, 128, 64, 1, (40,), (40,)),        # blocks of the two branches in different slabs
]
