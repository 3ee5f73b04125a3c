"""CPU check that the cases of tests/test_gpu_lora_linear_grad.py reach every branch of the host-side planners of the linear LoRA
factor gradients (tests/lora_linear_plan.py) at 132 SMs (H100 SXM) and at 114 SMs (H100 PCIe): both clamps of the pair's SM split and
its proportional middle, one row split, several, and the floor at one when a problem has more 128-column chunks than CTAs, part-filled
last chunks, the M tails, and the rank-column layouts of the block tables."""
import pytest

from lora_linear_plan import (H100_PCIE_SMS, H100_SMS, TWO_INPUT_CASES, branches, grad_cases, grad_plan, lora_layout, pair_cases,
                              pair_plan, problem_plan, slabs)


def test_planners_follow_the_kernels_documented_choices():
    # SD1.5 q|k|v at batch 2: 3 chunks of x against 8 of dY -> t0 = round(132 * 3 / 11) = 36; 64 tiles in 11 splits of 6
    p = pair_plan(8192, 320, 960, 132)
    assert p["t0"] == 36 and p["clamp"] == "none"
    assert {k: p["down"][k] for k in ("n_tiles", "splits", "tiles_per_cta", "ctas")} == {"n_tiles": 3, "splits": 11, "tiles_per_cta": 6,
                                                                                          "ctas": 33}
    assert {k: p["up"][k] for k in ("n_tiles", "splits", "ctas")} == {"n_tiles": 8, "splits": 11, "ctas": 88}
    # t0 rounds half up (132 * 2 / 7 = 37.7 -> 38; 132 / 264 = 0.5 -> 1, 132 * 263 / 264 = 131.5 -> 132), clamped at either end
    assert pair_plan(1, 128 * 2, 128 * 5, 132)["t0"] == 38
    assert pair_plan(1, 128, 128 * 263, 132)["clamp"] == "none" and pair_plan(1, 128, 128 * 264, 132)["clamp"] == "low"
    assert pair_plan(1, 128 * 262, 128, 132)["clamp"] == "none" and pair_plan(1, 128 * 263, 128, 132)["clamp"] == "high"
    # the split never exceeds the tiles, and a floored problem keeps one split per chunk
    assert problem_plan(16513, 0, 320, 132) == {"n_tiles": 3, "splits": 44, "tiles_per_cta": 3, "ctas": 132, "kind": "several",
                                                "part_chunk": True}
    assert problem_plan(300, 0, 128 * 200, 131)["ctas"] == 200
    assert grad_plan(77, 0, 128 * 133 + 64, 132)["kind"] == "floor"


@pytest.mark.parametrize("sms", [H100_SMS, H100_PCIE_SMS])
def test_pair_cases_reach_every_branch(sms):
    seen = set()
    for name, M, K, N, blocks, want in pair_cases(sms):
        p = pair_plan(M, K, N, sms)
        assert branches(want, p) == want, f"{name} at {sms} SMs: {branches(want, p)} != {want}"
        seen.add(("clamp", p["clamp"]))
        for prob in ("down", "up"):
            seen.add(("row splits", p[prob]["kind"]))
            if p[prob]["part_chunk"]:
                seen.add("part-filled last chunk")
        if M <= 128:
            seen.add("M <= 128")
        seen.add(("M", M if M in (1, 77, 127, 129) else "> 16384" if M > 16384 else "other"))
        if M > 128:
            seen.add(("M % 128", M % 128))
    want = {("clamp", "low"), ("clamp", "high"), ("clamp", "none"), ("row splits", "one"), ("row splits", "several"),
            ("row splits", "floor"), "part-filled last chunk", "M <= 128", ("M", 1), ("M", 77), ("M", 127), ("M", 129), ("M", "> 16384")}
    assert want <= seen, want - seen
    assert {1, 77 % 128, 127} <= {M % 128 for _, M, *_ in pair_cases(sms)}


@pytest.mark.parametrize("sms", [H100_SMS, H100_PCIE_SMS])
def test_grad_cases_reach_every_branch(sms):
    seen = set()
    for name, M, n_begin, n_end, ldx, blocks, want in grad_cases(sms):
        p = grad_plan(M, n_begin, n_end, sms)
        assert branches(want, p) == want, f"{name} at {sms} SMs: {branches(want, p)} != {want}"
        assert n_begin % 8 == 0 and ldx % 8 == 0 and n_end <= ldx
        assert all(n_begin <= lo < hi <= n_end for _, lo, hi, _ in blocks)
        seen.add(("row splits", p["kind"]))
        seen.add(("transpose_out", tuple(sorted({t for *_, t in blocks}))))
        if n_begin > 0:
            seen.add("n_begin > 0")
        if p["part_chunk"]:
            seen.add("part-filled last chunk")
        covered = set().union(*(range(lo, hi) for _, lo, hi, _ in blocks))
        if len(covered) < n_end - n_begin:
            seen.add("X columns of no block inside [n_begin, n_end)")
        if ldx > n_end:
            seen.add("X columns past n_end")
    want = {("row splits", "one"), ("row splits", "several"), ("row splits", "floor"), ("transpose_out", (0, 1)), "n_begin > 0",
            "part-filled last chunk", "X columns of no block inside [n_begin, n_end)", "X columns past n_end"}
    assert want <= seen, want - seen


def test_tables_reach_every_layout():
    seen = set()
    for name, M, K, N, blocks, _ in pair_cases():
        ranks = [r for r, _, _ in blocks]
        c0s, r_tot, R = lora_layout(ranks)
        assert all(o0 + out <= N for _, o0, out in blocks)
        if len(blocks) == 3 and [o0 for _, o0, _ in blocks] == [0, N // 3, 2 * N // 3]:
            seen.add("q|k|v: n_lo 0 / C / 2C")
        if len(blocks) == 1 and blocks[0][1] > 0 and blocks[0][1] + blocks[0][2] < N:
            seen.add("one block over part of dY")
        if any(c0 % 64 + r < 64 for c0, r in zip(c0s, ranks)) and len(blocks) > 1 and r_tot > sum(ranks):
            seen.add("unused slab columns between blocks")
        if r_tot % 64 and len(slabs(ranks)) == 1 and len(blocks) > 1:
            seen.add("unused slab columns after the blocks")
        for _, pieces in slabs(ranks):
            if len(pieces) > 8:
                seen.add("more than 8 pieces in one slab: two launches")
        if any(r > 64 for r in ranks):
            seen.add(("one block over two slabs, rank", max(ranks)))
        seen.add(("R", R))
    for M, K0, K1, N, blocks in TWO_INPUT_CASES:
        seen.add("two inputs")
        if len(slabs([r for r, _, _ in blocks])) > 1:
            seen.add("two inputs, two slabs")
    want = {"q|k|v: n_lo 0 / C / 2C", "one block over part of dY", "unused slab columns between blocks", "unused slab columns after the blocks",
            "more than 8 pieces in one slab: two launches", ("one block over two slabs, rank", 80), ("one block over two slabs, rank", 128),
            ("R", 64), ("R", 128), ("R", 192), "two inputs", "two inputs, two slabs"}
    assert want <= seen, want - seen
