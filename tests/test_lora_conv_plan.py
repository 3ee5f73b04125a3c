"""CPU check that the cases of tests/test_gpu_lora_conv_edges.py reach every branch of the host-side planners of the Conv2d LoRA
path (tests/lora_conv_plan.py): each convolution box geometry, each K-split branch with a LoRA segment, each shape of the dW_down
grid, each rank-column layout, and a DreamArtist++ tile that holds both batch halves."""
from lora_conv_plan import (CASES, DAPP_CASES, UP_CASES, conv_box, dapp_straddles, klast, lora_grad_plan, lora_layout, slabs,
                            split_plan, tile_n)


def plan(case):
    B, H, W, Cin, Cout, s, ranks = case
    _, r_tot, R = lora_layout(ranks)
    return conv_box(B, H, W, s), split_plan(B, H, W, Cin, Cout, s, R, r_tot), lora_grad_plan(B, H, W, Cin, s)


def test_planners_follow_the_kernels_documented_choices():
    # the 8x8 level: BN 160, 8 output tiles, 9 * 20 + 1 = 181 k-blocks -> 16 splits of 12, the LoRA k-block alone in the last
    assert tile_n(1280) == 160
    assert split_plan(2, 8, 8, 1280, 1280, 1, 64, 16) == {"ctas": 8, "total_kb": 181, "splits": 16, "branch": "wave",
                                                          "kb_per_split": 12, "lora_split": 15, "lora_alone": True}
    assert conv_box(1, 128, 128, 1) == {"bw": 128, "bh": 1, "bnimg": 1, "tiles_w": 1, "tiles_h": 128, "m_tiles": 128}
    assert conv_box(3, 2, 2, 1)["bnimg"] == 32 and conv_box(3, 2, 2, 1)["m_tiles"] == 1
    assert lora_grad_plan(1, 128, 128, 320, 1) == {"col_chunks": 3, "part_chunk": True, "splits": 43, "tiles_per_cta": 3}
    assert lora_layout((40, 40, 40)) == ([0, 64, 128], 168, 192)
    assert lora_layout((80,)) == ([0], 80, 128)
    assert [klast(r) for r in (4, 12, 16, 20, 36, 64, 80, 168)] == [1, 1, 1, 2, 3, 4, 1, 3]


def test_forward_cases_reach_every_box_and_split_branch():
    seen = set()
    for case in CASES:
        B, H, W, Cin, Cout, s, ranks = case
        box, sp, _ = plan(case)
        seen.add(("stride", s))
        if box["bw"] == 128:
            seen.add(("bw 128, tiles_w", box["tiles_w"]))
        elif box["bnimg"] == 1:
            seen.add("bw < 128, one image a tile")
        elif B % box["bnimg"]:
            seen.add("several images a tile, the last tile part-filled")
        seen.add(("split", "none" if sp["splits"] == 1 else "two halves" if sp["branch"] == "halves" else "many"))
        r_tot = lora_layout(ranks)[1]
        if sp["splits"] > 1:
            seen.add(("LoRA k-block", "alone in its split" if sp["lora_alone"] else "shares its split"))
            if r_tot % 16:
                seen.add("split with a partial last LoRA k-step")
        seen.add(("klast", klast(r_tot)))
        seen.add(("Cout % 64 == 0 (w_tiled)", Cout % 64 == 0))
    want = {("stride", 1), ("stride", 2), ("bw 128, tiles_w", 1), ("bw 128, tiles_w", 2), "bw < 128, one image a tile",
            "several images a tile, the last tile part-filled", ("split", "none"), ("split", "two halves"), ("split", "many"),
            ("LoRA k-block", "alone in its split"), ("LoRA k-block", "shares its split"), "split with a partial last LoRA k-step",
            ("klast", 1), ("klast", 2), ("klast", 3), ("klast", 4), ("Cout % 64 == 0 (w_tiled)", True)}
    assert want <= seen, want - seen


def test_gradient_cases_reach_every_chunk_and_row_split():
    seen = set()
    for case in CASES:
        B, H, W, Cin, Cout, s, ranks = case
        box, _, g = plan(case)
        seen.add(("col_chunks", min(g["col_chunks"], 3)))
        if g["part_chunk"]:
            seen.add("part-filled column chunk")
            if s == 2 and Cin % 128 == 64:
                seen.add("stride 2: discarded phase half")
        seen.add(("row splits", "1" if g["splits"] == 1 else "> 1"))
        seen.add(("box", "bw 128" if box["bw"] == 128 else "bnimg > 1" if box["bnimg"] > 1 else "bw < 128"))
        seen.add(("grad stride", s))
        _, _, R = lora_layout(ranks)
        seen.add(("R", R))
        c0s, r_tot, _ = lora_layout(ranks)
        if r_tot > sum(ranks):
            seen.add("slab-alignment gap")
        if any(c0 > 0 for c0 in c0s):
            seen.add("c0 > 0")
        for _, pieces in slabs(ranks):
            if len(pieces) > 8:
                seen.add("more than 8 pieces in one slab")
            if any(cs > 0 for *_, cs in pieces):
                seen.add("piece at a column > 0 of its slab")
        if any(r > 64 for r in ranks):
            seen.add("one block over two slabs")
    want = {("col_chunks", 1), ("col_chunks", 2), ("col_chunks", 3), "part-filled column chunk", "stride 2: discarded phase half",
            ("row splits", "1"), ("row splits", "> 1"), ("box", "bw 128"), ("box", "bnimg > 1"), ("box", "bw < 128"),
            ("grad stride", 1), ("grad stride", 2), ("R", 64), ("R", 128), ("R", 192), "slab-alignment gap", "c0 > 0",
            "more than 8 pieces in one slab", "piece at a column > 0 of its slab", "one block over two slabs"}
    assert want <= seen, want - seen
    # dW_up: dY read in 128-column chunks, the last part-filled (320 = 2.5 x 128, 640 = 5 x 128), and a slab past the first
    assert {-(-N // 128) for _, N, _ in UP_CASES} == {3, 5} and any(N % 128 for _, N, _ in UP_CASES)
    assert any(len(slabs(r)) > 1 for *_, r in UP_CASES) and any(len(p) > 8 for *_, r in UP_CASES for _, p in slabs(r))


def test_dapp_cases_straddle_and_split_the_batch_halves():
    kinds = set()
    for B, H, W, Cin, Cout, s, rn, rp in DAPP_CASES:
        assert B % 2 == 0
        kinds.add(("stride", s))
        kinds.add("a tile holds both halves" if dapp_straddles(B, H, W, s) else "halves in separate tiles")
        c0s, _, R = lora_layout(rn + rp)
        if min(c0s[len(rn):]) >= 64:
            kinds.add("branches in different slabs")
    assert kinds >= {("stride", 1), ("stride", 2), "a tile holds both halves", "halves in separate tiles", "branches in different slabs"}
