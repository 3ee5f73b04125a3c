"""CPU check that the cases of tests/test_gpu_norm_wgrad_edges.py reach every branch of the host-side planners they restate
(tests/norm_wgrad_plan.py): each GroupNorm path and cluster size, each LayerNorm instantiation, each weight-gradient tile geometry."""
from norm_wgrad_plan import (AFFINE_CASES, COLSUM_CASES, CONV_WGRAD_CASES, GN_BATCH_CASES, GN_CASES, GN_OFFSET_SHAPES, GN_TWO_PASS_CASES,
                             LN_CASES, REPACK_JOBS, SMALL_LINEAR_CASES, WGRAD_CASES, conv_wgrad_plan, gn_plan, ln_plan, repack_paths,
                             small_linear_dx_plan, wgrad_plan)


def test_planners_follow_the_kernels_documented_choices():
    # SD1.5 64x64 level: single pass, 8 CTAs of 512 pixels x 40 channels; 16384 pixels: the forward slab (160 KB) fits, the backward's
    # does not; a concatenation boundary inside a channel block takes gn8; two channels per group take the pair kernels
    assert gn_plan(4096, 320, 0, 32, True) == {"path": "gnf", "cg": 10, "S": 8, "CB": 40, "V": 5, "gpb": 4, "lanes": 64, "P": 512}
    assert gn_plan(16384, 320, 0, 32, False)["path"] == "gnf" and gn_plan(16384, 320, 0, 32, True)["path"] == "gn8"
    assert gn_plan(1024, 640, 320, 32, False)["path"] == "gn8"
    assert gn_plan(1024, 64, 0, 32, False)["path"] == "gn"
    assert gn_plan(4096, 320, 0, 32, False, two_pass=True)["path"] == "gn8"
    assert ln_plan(16384, 320) == {"nvpl": 2, "pipe": True, "rpw": 8, "last_rows": 8}
    assert wgrad_plan(16384, 320, 320) == {"sn": 128, "splits": 26, "max_splits": 30, "tiles_per_cta": 5}
    assert conv_wgrad_plan(1, 128, 128, 1) == {"bw": 128, "bh": 1, "bnimg": 1}


def test_groupnorm_cases_reach_every_path_and_cluster_size():
    seen = set()
    for B, HW, C1, C2, _ in GN_CASES + [(B, HW, C1, C2, True) for B, HW, C1, C2 in GN_OFFSET_SHAPES]:
        for bwd in (False, True):
            p = gn_plan(HW, C1, C2, 32, bwd)
            seen.add(("path", p["path"]))
            if p["path"] == "gnf":
                seen |= {("S", p["S"]), ("CB", p["CB"]), ("gpb", p["gpb"]), ("lanes", p["lanes"])}
            if p["path"] == "gn8" and C2 and C1 % p["cg"]:
                seen.add("gn8 concatenation inside a group")
            if p["path"] == "gn":
                seen.add(("gn cg", p["cg"]))
        if gn_plan(HW, C1, C2, 32, False)["path"] == "gnf" and gn_plan(HW, C1, C2, 32, True)["path"] == "gn8":
            seen.add("mixed" if not C2 else "mixed concatenated")
        seen.add(("B", B))
    want = {("path", "gnf"), ("path", "gn8"), ("path", "gn"), ("S", 1), ("S", 2), ("S", 4), ("S", 8), ("CB", 40), ("CB", 80),
            ("CB", 120), ("gpb", 1), ("gpb", 2), ("gpb", 4), ("lanes", 64), ("lanes", 32), "gn8 concatenation inside a group",
            ("gn cg", 2), ("gn cg", 4), "mixed", "mixed concatenated", ("B", 1), ("B", 3)}
    assert want <= seen, want - seen
    assert {gn_plan(HW, C1, C2, 32, False)["path"] for _, HW, C1, C2 in GN_OFFSET_SHAPES} == {"gnf", "gn8", "gn"}
    # the forced two-pass leg covers the gnf shapes with every cluster size
    assert {gn_plan(c[1], c[2], c[3], 32, False)["S"] for c in GN_TWO_PASS_CASES} == {1, 2, 4, 8}
    assert all(gn_plan(c[1], c[2], c[3], 32, False, two_pass=True)["path"] == "gn8" for c in GN_TWO_PASS_CASES)


def test_batch_invariance_cases_reach_every_groupnorm_path():
    seen = set()
    for B, HW, C1, C2, _ in GN_BATCH_CASES:
        assert B > 1
        f, b = gn_plan(HW, C1, C2, 32, False), gn_plan(HW, C1, C2, 32, True)
        seen |= {(f["path"], f.get("S")), (b["path"], b.get("S"))}
        if f["path"] != b["path"]:
            seen.add("mixed")
    assert seen >= {("gnf", 1), ("gnf", 2), ("gnf", 4), ("gnf", 8), ("gn8", None), ("gn", None), "mixed"}, seen


def test_layernorm_cases_reach_every_instantiation():
    plans = [ln_plan(M, C) for M, C in LN_CASES]
    assert {p["nvpl"] for p in plans if not p["pipe"]} == set(range(1, 9))
    assert {p["nvpl"] for p in plans if p["pipe"]} == {1, 2}
    assert any(p["pipe"] and p["last_rows"] < p["rpw"] for p in plans)            # the last warp of the pipelined variant is short
    assert any(not p["pipe"] and p["rpw"] > 1 and p["last_rows"] < p["rpw"] for p in plans)
    assert any(not p["pipe"] and p["rpw"] >= 3 for p in plans)                     # many rows per warp, wide rows


def test_wgrad_cases_reach_every_tile_geometry():
    plans = [wgrad_plan(M, j, n) for M, j, n in WGRAD_CASES]
    assert {p["sn"] for p in plans} == {64, 128}
    assert any(j % wgrad_plan(M, j, n)["sn"] for M, j, n in WGRAD_CASES)          # a ragged j tile
    assert any(n % 128 and n > 128 for _, _, n in WGRAD_CASES)                    # a ragged n tile
    assert {M % 128 for M, _, _ in WGRAD_CASES} >= {1, 127}                       # one-row tails, one row short of a tile
    assert any(p["splits"] == 1 for p in plans) and any(p["splits"] > 1 for p in plans)
    assert any(p["splits"] == p["max_splits"] == 2 * 132 for p in plans)          # the maximum row split: one tile per CTA
    geos = {(tuple(conv_wgrad_plan(B, H, W, s).values()), s) for B, H, W, _, _, s in CONV_WGRAD_CASES}
    bn = {g[0][2] for g in geos}
    assert bn == {1, 2, 8, 32, 128}
    assert {s for g, s in geos if g[1] == 1 and g[2] == 1} == {1, 2}              # 128-wide rows, stride 1 and 2
    assert any(g[1] > 1 and g[2] == 1 for g, _ in geos)                           # several rows per tile
    assert any(B % conv_wgrad_plan(B, H, W, s)["bnimg"] for B, H, W, _, _, s in CONV_WGRAD_CASES)   # a part-filled image tile
    # stride 2 from 128-, 64- and 16-wide inputs, with a Cin that is not a multiple of 128 (the phase-overlap case) and Cin 128
    s2 = [(W, Cin) for _, _, W, Cin, _, s in CONV_WGRAD_CASES if s == 2]
    assert {W for W, _ in s2} >= {128, 64, 16} and {Cin % 128 for _, Cin in s2} == {0, 64}
    assert {Cout for *_, Cout, _ in CONV_WGRAD_CASES} >= {8, 64, 320, 336}


def test_repack_jobs_reach_every_kind_and_fallback():
    seen = {(k, p) for k, *rest in REPACK_JOBS for p in repack_paths(k, *rest)}
    assert seen >= {(0, "rows vector"), (0, "rows scalar"), (0, "cols vector"), (0, "cols scalar"), (0, "row tile tail"), (0, "o0 > 0"),
                    (1, "flip"), (1, "no flip"), (1, "Cout tail"), (1, "Cin tail"), (2, "copy"), (3, "rows vector"), (3, "rows scalar"),
                    (3, "row tile tail")}, seen


def test_small_linear_cases_reach_n_chunk_growth():
    plans = [small_linear_dx_plan(M, N, K) for M, N, K, _ in SMALL_LINEAR_CASES]
    assert [p["n_chunk"] for p in plans] == [512, 1024, 512]
    assert max(p["row_blocks"] for p in plans) > 1


def test_reduction_cases_reach_chunk_halving_and_tails():
    assert any(HW > 1024 and g for _, HW, _, _, g, _ in AFFINE_CASES)
    assert any(C1 % 64 and C2 for _, _, C1, C2, _, _ in AFFINE_CASES)            # concatenation boundary inside a 64-channel block
    assert {g for *_, g, _ in AFFINE_CASES} == {0, 32}
    assert any(rpg > 512 and rpg % 2 == 0 for _, _, _, rpg, _ in COLSUM_CASES)
    assert any(rpg > 512 and rpg % 2 for _, _, _, rpg, _ in COLSUM_CASES)
    assert any(ld > N for _, N, ld, _, _ in COLSUM_CASES) and any(s != 1 for *_, s in COLSUM_CASES)
    assert any(N % 64 for _, N, _, _, _ in COLSUM_CASES)
