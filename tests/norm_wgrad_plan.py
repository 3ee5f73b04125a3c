"""Host-side planners of the normalisation and weight-gradient kernels, restated in Python (as `tile_n` in test_gpu_edges.py restates
`pick_bn`), and the case lists of tests/test_gpu_norm_wgrad_edges.py.  tests/test_norm_wgrad_plan.py checks on the CPU that the
cases reach every branch of every planner; the GPU tests use the same functions to name the path a case takes and its tiles.

  gn_plan       gnf_plan + gn_geometry (norms.cu): single-pass cluster kernel `gnf` (S CTAs per image and channel block of CB
                channels, V 16-byte vectors per pixel row, 64 or 32 pixel lanes), two-pass 8-vector kernels `gn8`, two-pass pair kernels `gn`
  ln_plan       launch_layernorm (norms.cu): NVPL 16-byte vectors per lane, the software-pipelined variant, rows per warp
  wgrad_plan    run_wgrad (wgrad.cu): S-column tile SN and the number of row splits
  conv_box      plan_conv_box (host_util.cu): the 128-pixel box bw x bh x bnimg images of hcp_wgrad_conv3x3_bf16, which every 3x3
                convolution kernel shares; restated once, in tests/lora_conv_plan.py
"""
import math

from lora_conv_plan import conv_box  # noqa: F401

H100_SMS = 132          # H100 SXM; the GPU tests re-plan with the live SM count


def gn_plan(HW, C1, C2, G, bwd, two_pass=False):
    C = C1 + C2
    cg = C // G
    vec8 = cg >= 8 and C1 % 8 == 0 and C2 % 8 == 0 and C // 8 <= 1024
    two = {"path": "gn8" if vec8 else "gn", "cg": cg}
    if two_pass or cg < 8 or cg % 2 or C1 % 8 or C2 % 8:
        return two
    CB = cg // math.gcd(cg, 8) * 8
    if C % CB or (C2 > 0 and C1 % CB):
        return two
    V, gpb = CB // 8, CB // cg
    lanes = 64 if V <= 5 else 32
    if V * lanes > 512 or gpb > 8 or CB > 256:
        return two
    S = 1
    while S < 8 and HW % (2 * S) == 0 and HW // (2 * S) >= 64:
        S *= 2
    P = HW // S
    if P * CB * 2 * (2 if bwd else 1) > 180 * 1024:
        return two
    RB = min(P, 256)
    while RB >= 8 and (P % RB or RB % 8):
        RB -= 1
    if RB < 8:
        return two
    return {"path": "gnf", "cg": cg, "S": S, "CB": CB, "V": V, "gpb": gpb, "lanes": lanes, "P": P}


def ln_plan(M, C, sms=H100_SMS):
    wave = sms * 2 * 8
    rpw = min(32, max(1, -(-M // wave)))
    nvpl = (C // 8 + 31) // 32
    warps = -(-M // rpw)
    return {"nvpl": nvpl, "pipe": rpw >= 3 and nvpl <= 2, "rpw": rpw, "last_rows": M - (warps - 1) * rpw}


def wgrad_plan(M, j_cols, n_cols, sms=H100_SMS):
    sn = 128 if j_cols > 64 else 64
    out_tiles = -(-n_cols // 128) * -(-j_cols // sn)
    total = -(-M // 128)
    splits = min(total, max(1, -(-2 * sms // out_tiles)))
    per = -(-total // splits)
    return {"sn": sn, "splits": -(-total // per), "max_splits": min(total, -(-2 * sms // out_tiles)), "tiles_per_cta": per}


def small_linear_dx_plan(M, N, K):
    """n_chunk of hcp_small_linear_bwd_f32's dx kernel (wgrad.cu): output columns per block, doubled while the grid exceeds 592 blocks
    per 16-row block."""
    kb = -(-K // 128)
    n_chunk = 512
    while n_chunk < N and kb * -(-N // n_chunk) > 592:
        n_chunk *= 2
    return {"n_chunk": n_chunk, "row_blocks": -(-M // 16)}


# ---------------------------------------------------------------------------------------------------------------------------------
# case lists
# ---------------------------------------------------------------------------------------------------------------------------------
# GroupNorm (B, HW, C1, C2, silu) with 32 groups.  SD / SDXL widths: 320 / 640 / 1280 (CB 40, 4 / 2 / 1 groups per block), 960 and
# 1920 (CB 120: 15 vectors, 32 lanes, a vector straddling two groups), 2560 (CB 80); HW 64 / 128 / 256 / >= 512 give S = 1 / 2 / 4 / 8
GN_CASES = [
    (1, 64, 1280, 0, True), (3, 64, 2560, 0, False), (2, 64, 1280, 1280, True),           # 8x8 level / mid block: S = 1
    (3, 128, 640, 0, True), (1, 128, 960, 0, False),                                        # S = 2 (an 8x16 map)
    (1, 256, 320, 320, True), (3, 256, 1920, 0, True),                                      # S = 4
    (1, 1024, 320, 0, True), (2, 1024, 640, 0, False), (1, 4096, 960, 0, True),             # S = 8
    (2, 256, 1280, 640, True), (1, 1024, 640, 320, False),                                  # gn8: concatenation inside a group
    (3, 100, 64, 0, True), (1, 256, 128, 0, False), (2, 64, 64, 64, True),                  # pair kernels: 2 / 4 channels per group
    (1, 16384, 320, 0, True), (1, 16384, 320, 320, True), (1, 16384, 640, 320, False),      # fwd gnf / bwd gn8; 640 + 320: gn8 both
]
# the same shapes with the two-pass kernels forced (HCP_GN_TWO_PASS): the gnf cases of GN_CASES
GN_TWO_PASS_CASES = [c for c in GN_CASES if gn_plan(c[1], c[2], c[3], 32, False)["path"] == "gnf"]
# batch invariance (image 1 of 3 against the same image alone) on every path: gnf with S = 1 / 2 / 4 / 8, gn8 with a concatenation
# inside a group, the pair kernels, and the 16384-pixel shape whose forward is gnf and backward gn8
GN_BATCH_CASES = [c for c in GN_CASES if c[0] == 3] + [(3, 1024, 320, 0, True), (3, 256, 1280, 640, True), (3, 16384, 320, 0, True)]
# offset stress: per-group means of 0, 8 and 64 standard deviations on each path
GN_OFFSET_SHAPES = [(2, 1024, 320, 0), (2, 256, 1280, 640), (2, 256, 128, 0)]
GN_OFFSETS = [0.0, 8.0, 64.0]

# LayerNorm (M, C): NVPL 1-8, the pipelined variant at the 64x64 level (M 16384, C 320) and with a short last warp (M 16389), a row
# tail in the plain variant with two rows per warp, and a plain variant with many rows per warp (C 1280)
LN_CASES = [(300, 8), (300, 40), (300, 320), (300, 768), (300, 1024), (300, 1280), (300, 1536), (300, 1792), (300, 2048),
            (16384, 320), (16389, 320), (16389, 40), (4001, 768), (16384, 1280), (77, 2048)]

# linear weight gradient (M, j_cols, n_cols): SN 64 / 128 with ragged j tiles, M tails of one row, the maximum row split
WGRAD_CASES = [(1, 8, 8), (127, 64, 72), (129, 72, 320), (129, 320, 8), (16384, 320, 320), (16384, 8, 72), (16384, 72, 8),
               (127, 320, 72), (1, 72, 320), (16384, 64, 320), (33792, 64, 72)]
# 3x3 weight gradient (B, Hin, Win, Cin, Cout, stride)
CONV_WGRAD_CASES = [
    (1, 128, 128, 320, 320, 1), (1, 4, 256, 64, 64, 1),                 # one 128-pixel row (SDXL top level), two boxes per row
    (2, 64, 64, 320, 336, 1),                                           # several rows (64x64 level)
    (3, 8, 8, 640, 64, 1), (5, 4, 4, 128, 8, 1), (33, 2, 2, 64, 64, 1), (130, 1, 1, 64, 336, 1),     # 2 / 8 / 32 / 128 images a tile
    (1, 8, 256, 320, 64, 2), (1, 128, 128, 320, 320, 2), (2, 64, 64, 128, 64, 2), (3, 16, 16, 320, 336, 2), (2, 16, 16, 128, 8, 2),
]

# affine gradients (B, HW, C1, C2, groups, silu): GroupNorm (groups 32) incl. straddling vectors and concatenations, rows per image
# above 1024 (chunk halving: 4096 -> 1024, 2052 -> 1026 -> 513), LayerNorm rows (groups 0)
AFFINE_CASES = [(2, 256, 320, 0, 32, True), (2, 64, 1280, 640, 32, True), (3, 1024, 640, 320, 32, False), (1, 4096, 960, 0, 32, True),
                (2, 2052, 200, 120, 32, False), (1, 3000, 320, 0, 0, False), (1, 16384, 320, 0, 0, False), (4, 77, 768, 0, 0, False)]
# repack jobs (kind, rows, K, o0, n_tot, flip) of one hcp_repack_weights launch: a q|k|v group with K not a multiple of 4 (scalar
# rows) of which two hosts are written; a 128-row host at o0 128 (vector rows and columns); a k|v host with K 72 and a 100-row tail
# (vector columns, scalar tail); n_tot | o0 odd (scalar columns); 3x3 weights with Cout not a multiple of 16 and Cin not a multiple of
# 64, flipped (stride 1) and not (stride 2); a bias slice; time-embedding rows with and without the vector path
REPACK_JOBS = [(0, 67, 70, 67, 201, 0), (0, 67, 70, 134, 201, 0), (0, 128, 320, 128, 384, 0), (0, 100, 72, 100, 200, 0),
               (0, 65, 64, 65, 130, 0), (1, 24, 72, 0, 0, 1), (1, 40, 136, 0, 0, 0), (1, 320, 320, 0, 0, 1),
               (2, 100, 1, 37, 0, 0), (3, 50, 66, 20, 0, 0), (3, 64, 128, 64, 0, 0)]


def repack_paths(kind, rows, K, o0, n_tot, flip):
    """Store paths of repack_kernel (wgrad.cu) one job takes."""
    if kind == 2:
        return {"copy"}
    if kind == 1:
        return {"flip" if flip else "no flip"} | ({"Cout tail"} if rows % 16 else set()) | ({"Cin tail"} if K % 64 else set())
    out = {"rows vector" if K % 4 == 0 else "rows scalar"} | ({"row tile tail"} if rows % 64 else set())
    if kind == 0:
        vec = (n_tot | o0) % 4 == 0
        out |= {"cols vector"} if vec and rows >= 4 else set()
        out |= {"cols scalar"} if not vec or rows % 4 else set()
        out |= {"o0 > 0"} if o0 else set()
    return out


# small fp32 linear backward (M, N, K, with dW / db): several 16-row blocks (M 17, 64); (64, 40960, 1280) is the case whose dx grid
# doubles n_chunk (10 k-blocks x 80 chunks of 512 > 592) -- dx only: a dW reference of 40960 x 1280 adds nothing the others miss
SMALL_LINEAR_CASES = [(17, 5120, 320, True), (64, 40960, 1280, False), (3, 1280, 2816, True)]

# column sums (M, N, ld, rows_per_group, scale): chunk halving (4096 -> 512), an odd group of 1025 rows, N tails of a 64-column block
COLSUM_CASES = [(16384, 320, 320, 0, 1.0), (3 * 4096, 320, 384, 4096, 0.25), (3 * 1025, 200, 256, 1025, 1.0), (300, 8, 8, 100, 0.5),
                (2 * 77, 1280, 1280, 77, 1.0)]
