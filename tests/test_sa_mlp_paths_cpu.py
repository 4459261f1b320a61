"""The GPU tests of the fused shared-MLP + max-pool node reach every small-K instance, every channel width, every
backward branch and every grid-strided row-kernel loop.

tests/sa_mlp_paths.py restates the selection rules of sa_mlp.py and the grids of csrc/sa_mlp_kernels.cu; this maps the
case lists of test_sa_mlp_edges_gpu.py through them.  Removing a case, or moving a rule in the sources without a GPU
case that runs the new side, fails here, without a GPU."""
import sa_mlp_paths as P
import test_sa_mlp_edges_gpu as E


def _node_cases():
    return [dict(cin=s[0], widths=s[1:], b=b, npoint=n, group=g, x_grad=xg, ties=t)
            for s, b, n, g, xg, t in E.NODE_CASES]


def test_restated_rules_on_known_shapes():
    # the step's pre-encoder: xyz through the small-K instance, 256 wide at group 64 -> POOLED_PRE
    assert P.applicable(3, [64, 128, 256], 64, False)
    assert P.small_k(3) == 3 and P.small_k(64) is None
    assert P.backward_branches(3, [64, 128, 256], 64) == {"small_k", "pooled_pre"}
    assert P.backward_branches(3, [128], 16) == {"single_block_expand"}
    assert P.backward_branches(64, [128, 32], 64) == {"expand"}
    assert P.backward_branches(64, [128], 96) == {"expand"}             # 96 tiles 32 rows but not 128
    # 8 x 2048 x 64 rows at 64 channels: 16 row slots, 528 blocks, a grid-stride loop of 125 steps
    assert P.slots(64) == 16 and P.grid_for(8 * 2048 * 64, 64) == 528 and P.strided(8 * 2048 * 64, 64)
    assert P.slots(1024) == 1 and P.slots(4) == 256
    assert P.grid_for(2, 1024) == 2 and not P.strided(528 * 4, 256) and P.strided(528 * 4 + 1, 256)
    assert P.maxpool_grid(16384) == 1056 and P.maxpool_grid(100) == 100
    # declines
    assert not P.applicable(3, [64], 16, True)                          # no input gradient from the tiny-K layer
    assert not P.applicable(72, [64], 16, False)
    assert not P.applicable(64, [96, 128], 16, False)                   # non-last width not a multiple of 64
    assert not P.applicable(3, [64], 257, False)
    assert not P.applicable(3, [12], 16, False)                         # 12 / 4 does not divide 256
    # GEMM layers wider than 256: their column statistics do not fit beside the GEMM's stages
    assert not P.applicable(64, [512, 1024], 32, True) and not P.applicable(3, [64, 512], 32, False)
    assert P.applicable(3, [1024], 7, False)


def test_node_cases_are_applicable_and_reach_every_instance_and_branch():
    cases = _node_cases()
    for c in cases:
        assert P.applicable(c["cin"], c["widths"], c["group"], c["x_grad"]), c
    assert {P.small_k(c["cin"]) for c in cases} >= set(range(1, 9))
    branches = set().union(*(P.backward_branches(c["cin"], c["widths"], c["group"]) for c in cases))
    assert branches == {"single_block_expand", "pooled_pre", "expand", "small_k"}
    # POOLED_PRE at every group that tiles the 128-row blocks, each with an odd group count
    pre = {c["group"] for c in cases if "pooled_pre" in P.backward_branches(c["cin"], c["widths"], c["group"])
           and (c["b"] * c["npoint"]) % 2}
    assert pre >= {32, 64, 128, 256}
    # the expand path at a group that tiles 32 rows but not 128, and at an odd group, under a GEMM layer
    expand = [c for c in cases if "expand" in P.backward_branches(c["cin"], c["widths"], c["group"])]
    assert {96, 7} <= {c["group"] for c in expand}
    # narrow last layers through the GEMMs
    assert {4, 32} <= {c["widths"][-1] for c in expand}
    # the widest last layers (2 row slots and 1), which only a small-K first layer reaches
    assert {512, 1024} <= {c["widths"][-1] for c in cases}
    assert any(c["ties"] for c in cases)
    # the step's configuration, and the use_color one, at group 64
    assert any(c["cin"] == 3 and list(c["widths"]) == [64, 128, 256] and c["group"] == 64 and not c["ties"]
               and c["b"] * c["npoint"] > P.MAXPOOL_BLOCKS and (c["b"] * c["npoint"]) % 2 for c in cases)
    assert any(c["cin"] == 6 and list(c["widths"]) == [64, 128, 256] and c["group"] == 64 for c in cases)


def test_row_kernel_cases_reach_every_width_and_grid_stride():
    launches = []
    for c in _node_cases():
        launches += P.node_launches(c["cin"], c["widths"], c["b"], c["npoint"], c["group"])
    # the isolated tests: statistics / reduce kernels over ROW_CASES, the max-pool over MAXPOOL_CASES
    for c, rows in E.ROW_CASES:
        launches += [(k, rows, c, P.strided(rows, c)) for k in ("stats", "reduce", "reduce_pooled", "linear_small_k",
                                                                "bwd_small_k")]
    for c, groups, _ in E.MAXPOOL_CASES:
        launches.append(("maxpool", groups, c, groups > P.maxpool_grid(groups)))
    for kernel in ("stats", "reduce", "reduce_pooled", "linear_small_k", "bwd_small_k", "maxpool"):
        mine = [(rows, c, s) for k, rows, c, s in launches if k == kernel]
        assert {c for _, c, _ in mine} == set(P.WIDTHS), kernel
        for width in P.WIDTHS:
            assert any(s for _, c, s in mine if c == width), (kernel, width)         # a second grid-stride step
            assert any(rows == 2 for rows, c, _ in mine if c == width) or kernel == "maxpool", (kernel, width)
    # row counts that are not a multiple of the slot count, wherever there is more than one slot
    for c in P.WIDTHS:
        if P.slots(c) > 1:
            assert any(rows % P.slots(c) for cc, rows in E.ROW_CASES if cc == c), c
    # the step's own shape: the max-pool grid strides over its 4095 groups
    assert any(k == "maxpool" and s and c == 256 for k, _, c, s in launches)
    assert set(E.OFFSET_RATIOS) >= {10, 30}


def test_sync_bn_and_colsum_cases_reach_every_width_and_grid_stride():
    """tests/test_sync_bn_gpu.py: coda_bn_rows_sums (bn_stats_partial_kernel on grid_for's grid) and coda_rows_colsum
    (colsum_partial_kernel on at most 132 blocks) at every width, with and without a second grid-stride step; the
    simulated ranks at every width; the GEMM partials of a plain first layer, of AFFINE_RELU layers, and of both the
    B-resident and the tiled grid"""
    import gemm_instances as G
    import test_sync_bn_gpu as S

    for cases, strided in ((S.SUMS_CASES, P.strided), (S.COLSUM_CASES, P.colsum_strided)):
        assert {c for c, _ in cases} == set(P.WIDTHS)
        for width in P.WIDTHS:
            mine = [rows for c, rows in cases if c == width]
            assert any(strided(rows, width) for rows in mine), width
            assert any(not strided(rows, width) for rows in mine), width
            assert 2 in mine, width
            if P.slots(width) > 1:
                assert any(rows % P.slots(width) for rows in mine), width
    # colsum: exactly a full capped grid, and one row past it
    for width in P.WIDTHS:
        full = P.COLSUM_BLOCKS * P.slots(width)
        assert {full, full + 1} <= {rows for c, rows in S.COLSUM_CASES if c == width}, width
        assert P.colsum_grid(full, width) == P.COLSUM_BLOCKS and not P.colsum_strided(full, width)
        assert P.colsum_strided(full + 1, width)
    assert P.colsum_grid(1 << 20, 64) == 132 and P.grid_for(1 << 20, 64) == P.MAX_BLOCKS
    # the step's pre-encoder row count at 64, 128 and 256 channels
    assert {(c, 8 * 2048 * 64) for c in (64, 128, 256)} <= set(S.SUMS_CASES)
    # simulated ranks: 2, 3 and 8 at every width, from row passes and from GEMM partials
    assert {w for w, *_ in S.RANK_CASES} == {2, 3, 8}
    for w in (2, 3, 8):
        assert {c for ww, src, c, _ in S.RANK_CASES if ww == w and src == "rows"} == set(P.WIDTHS)
        assert any(ww == w and src == "gemm" for ww, src, *_ in S.RANK_CASES)
    # GEMM partials
    resident = {G.gemm_a32(ns, m, n, k, False, mode, True)[1] for ns, m, n, k, mode in S.PARTIAL_CASES}
    assert resident == {True, False}
    assert {mode for *_, mode in S.PARTIAL_CASES} == {G.A32_PLAIN, G.A32_AFFINE_RELU}
    assert any(G.gemm_a32(ns, m, n, k, False, mode, True)[1] and mode == G.A32_AFFINE_RELU
               for ns, m, n, k, mode in S.PARTIAL_CASES)
    # the node on gloo ranks: statistics from a row pass (small-K first layer) and from GEMM partials
    assert {P.small_k(spec[0]) is None for spec, *_ in S.NODE_RANK_CASES} == {True, False}
    for spec, b, npoint, group, x_grad in S.NODE_RANK_CASES:
        assert P.applicable(spec[0], spec[1:], group, x_grad)
    # the masked encoder's interim MLP (259 -> 256 -> 256 -> 256) is declined by the fused node
    assert not P.applicable(S.ENC_DIM + 3, [256, 256, S.ENC_DIM], S.ENC_NSAMPLE, False)
