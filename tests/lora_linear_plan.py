"""Host-side planners of the linear LoRA factor gradients (hcp_lora_grad_pair and hcp_lora_grad in wgrad.cu), restated in Python, and
the case lists of tests/test_gpu_lora_linear_grad.py.  tests/test_lora_linear_plan.py checks on the CPU that the cases reach every
branch at 132 SMs (H100 SXM) and at 114 SMs (H100 PCIe); the GPU tests re-plan with the live SM count and assert the branches each
case was chosen for.

  problem_plan  lg_problem + split_rows: X columns [n_begin, n_end) in 128-column chunks, and `target // n_tiles` CTAs (at least one,
                at most one per 128-row tile) sharing the rows of each chunk
  pair_plan     hcp_lora_grad_pair: t0 = round(sms * ck / (ck + cn)) CTAs for dW_down (ck, cn: 128-column chunks of x and dY),
                clamped to [1, sms - 1], the other sms - t0 for dW_up
  grad_plan     hcp_lora_grad: one problem with a target of one wave (sms CTAs)

Blocks of a case are (rank, o0, out_dim) hosts side by side in the rank columns, placed by lora_layout (tests/lora_conv_plan.py)
as ops.lora_columns places them and cut into slab pieces by `slabs` as ops.lora_slabs cuts them.
"""
from lora_conv_plan import H100_SMS, lora_layout, slabs  # noqa: F401

H100_PCIE_SMS = 114


def problem_plan(M, n_begin, n_end, target):
    n_tiles = -(-(n_end - n_begin) // 128)
    total = -(-M // 128)
    want = target // n_tiles
    splits = min(max(want, 1), total)
    per = -(-total // splits)
    splits = -(-total // per)
    kind = "floor" if want < 1 else "one" if splits == 1 else "several"
    return {"n_tiles": n_tiles, "splits": splits, "tiles_per_cta": per, "ctas": n_tiles * splits, "kind": kind,
            "part_chunk": (n_end - n_begin) % 128 != 0}


def pair_plan(M, K, N, sms=H100_SMS):
    ck, cn = -(-K // 128), -(-N // 128)
    t0 = (sms * ck + (ck + cn) // 2) // (ck + cn)
    clamp = "low" if t0 < 1 else "high" if t0 > sms - 1 else "none"
    t0 = min(max(t0, 1), sms - 1)
    return {"t0": t0, "clamp": clamp, "down": problem_plan(M, 0, K, t0), "up": problem_plan(M, 0, N, sms - t0)}


def grad_plan(M, n_begin, n_end, sms=H100_SMS):
    return problem_plan(M, n_begin, n_end, sms)


def branches(want, plan):
    """The subset of `plan` a case's `want` names: {"clamp": ..., "down": kind, "up": kind} (pair) or {"kind": ...} (hcp_lora_grad)."""
    return {k: (plan[k]["kind"] if isinstance(plan[k], dict) else plan[k]) for k in want}


def hosts(n, ranks):
    """Equal hosts of n outputs each, one block per host: (rank, o0, out_dim) with o0 = 0, n, 2n, ..."""
    return tuple((r, i * n, n) for i, r in enumerate(ranks))


# ---------------------------------------------------------------------------------------------------------------------------------
# case lists
# ---------------------------------------------------------------------------------------------------------------------------------
def pair_cases(sms=H100_SMS):
    """(id, M, K, N, blocks, want) of the pair launch (x [M, K], dY [M, N]); the planner-edge cases derive K or N from `sms`."""
    return [
        # layer shapes of the real models (M = tokens of a batch of two unless noted)
        ("sd15_qkv", 2 * 4096, 320, 960, hosts(320, (8, 8, 8)), {}),          # 64x64 level: three blocks in one slab, n_lo 0 / 320 / 640
        ("sdxl_qkv", 2 * 1024, 1280, 3840, hosts(1280, (32, 32, 32)), {}),    # 32x32 level: the third block starts slab 1 (c0 64)
        ("sd15_to_kv", 77 * 2, 768, 640, hosts(320, (16, 16)), {}),          # to_k|to_v: x = the 768-wide CLIP-L context (77 rows an image)
        ("sdxl_to_kv", 77 * 4, 2048, 2560, hosts(1280, (16, 16)), {}),       # the 2048-wide SDXL context at batch 4
        ("sd15_ff_proj", 2 * 4096, 320, 2560, hosts(2560, (32,)), {}),        # GEGLU proj 320 -> 2560
        ("sdxl_ff_proj", 2 * 1024, 1280, 10240, hosts(10240, (32,)), {}),     # 1280 -> 10240: 10 chunks against 80, t0 = 15
        ("sd15_ff_out", 2 * 1024, 1280, 320, hosts(320, (16,)), {}),          # ff out 1280 -> 320 (32x32 level)
        ("sdxl_ff_out", 2 * 1024, 5120, 1280, hosts(1280, (64,)), {}),        # 5120 -> 1280, a full slab
        ("clip_l_qkv", 77 * 4, 768, 2304, hosts(768, (4, 4, 4)), {}),         # CLIP-L self-attention q|k|v at batch 4: M 308
        ("bigg_fc1", 77 * 3, 1280, 5120, hosts(5120, (8,)), {}),              # OpenCLIP-bigG mlp fc1 at batch 3: M 231
        ("clip_l_fc2", 77 * 2, 3072, 768, hosts(768, (8,)), {}),              # CLIP-L mlp fc2 at batch 2: M 154
        # planner edges
        ("t0_low", 77, 64, 128 * (2 * sms + 2), hosts(128 * (2 * sms + 2), (16,)),   # t0 rounds to 0 -> 1; dY has more chunks
         {"clamp": "low", "down": "one", "up": "floor"}),                             # than its sms - 1 CTAs: one split each
        ("t0_high", 129, 128 * (2 * sms + 2), 72, hosts(72, (16,)),                   # t0 rounds to sms -> sms - 1: dW_up gets one
         {"clamp": "high", "down": "floor", "up": "one"}),                            # CTA; N 72: a part-filled chunk
        ("m1", 1, 320, 320, hosts(320, (4,)), {"clamp": "none", "down": "one", "up": "one"}),          # one row
        ("m127", 127, 200, 72, hosts(72, (20,)), {"clamp": "none", "down": "one", "up": "one"}),       # part-filled chunks of both
        ("m129", 129, 1280, 320, hosts(320, (16,)), {"down": "several", "up": "several"}),             # two tiles, a one-row tail
        ("m16513", 16513, 640, 1280, hosts(640, (16, 16)), {"down": "several", "up": "several"}),      # > 16384 rows, tail 1
        ("uneven", 2048, 64, 10240, hosts(10240, (8,)), {"clamp": "none", "up": "one"}),     # t0 = 1 or 2 against 80
        # ranks and tables
        ("r20x3", 1000, 320, 960, hosts(320, (20, 20, 20)), {}),              # three blocks at c0 0 / 20 / 40, slab columns 60-63 unused
        ("r40x3", 1000, 320, 960, hosts(320, (40, 40, 40)), {}),              # one block per slab (c0 0 / 64 / 128): 24 unused columns each
        ("r80", 700, 256, 320, hosts(320, (80,)), {}),                        # two slabs: pieces of 64 and 16 rows, dst_ld 80
        ("r128", 700, 320, 256, hosts(256, (128,)), {}),                      # two slabs of 64 rows, dst_ld 128
        ("r4x9", 300, 320, 360, hosts(40, (4,) * 9), {}),                     # nine pieces in one slab: two launches; n_lo 40 apart
        ("k_only", 600, 320, 960, ((16, 320, 320),), {}),                     # only the k block of a q|k|v: n_lo 320, n_hi 640
    ]


def grad_cases(sms=H100_SMS):
    """(id, M, n_begin, n_end, ldx, blocks, want) of hcp_lora_grad alone: blocks (rank, n_lo, n_hi, transpose_out), c0 by lora_layout."""
    return [
        ("n_begin_mixed", 300, 72, 712, 720,                         # n_begin 72; transpose_out 0 and 1 in one table; X columns
         ((16, 72, 400, 0), (24, 200, 500, 1), (8, 640, 712, 1)),    # [500, 640) belong to no block
         {"kind": "several"}),
        ("floor", 77, 0, 128 * (sms + 1) + 64, 128 * (sms + 1) + 64,      # more 128-column chunks than SMs; the last part-filled
         ((16, 0, 128 * (sms + 1) + 64, 1),), {"kind": "floor"}),
        ("m1", 1, 8, 136, 144, ((4, 8, 136, 0), (4, 8, 136, 1)), {"kind": "one"}),                  # one row, the same product twice
        ("m16513", 16513, 0, 320, 320, ((64, 0, 320, 0),), {"kind": "several"}),                    # a full slab over 130 tiles
    ]


# two-input layers (M, K0, K1, N, blocks): the pair on input 0, hcp_lora_grad on input 1 at the destination offset K0
TWO_INPUT_CASES = [
    (2 * 1024, 1280, 640, 640, hosts(640, (16,))),                # SD1.5 up_blocks[2] conv_shortcut at 32x32: [1280 | 640] -> 640
    (2 * 4096, 640, 320, 320, ((40, 0, 320), (40, 0, 320))),     # up_blocks[3] at 64x64: [640 | 320] -> 320, two adapters, two slabs
]
