"""The GPU tests of the step's glue kernels reach every LayerNorm instance in every form, every BatchNorm width on both
sides of the grid stride, every dropout tail, every AdamW head / tail split and both Hungarian layouts and orientations.

tests/step_glue_paths.py restates the selection rules of csrc/detr_kernels.cu and csrc/step_kernels.cu; this maps the
case lists of test_step_glue_edges_gpu.py, test_detr_kernels_gpu.py and test_step_kernels_gpu.py through them.
Removing a case, or moving a rule in the sources without a GPU case that runs the new side, fails here, without a GPU.
It also checks the dropout twin itself against values worked out by hand."""
import numpy as np

import step_glue_paths as P
import test_detr_kernels_gpu as D
import test_step_glue_edges_gpu as E
import test_step_kernels_gpu as S


def _params(fn):
    """argument tuples of a test's @pytest.mark.parametrize"""
    (mark,) = [m for m in fn.pytestmark if m.name == "parametrize"]
    return [a if isinstance(a, tuple) else (a,) for a in mark.args[1]]


def _ln_launches():
    """-> {(form, nv, rows)} of every LayerNorm launch the GPU tests make"""
    out = set()
    for variant, nv, rows in E.LN_CASES:
        fwd = {"plain": "fwd", "pos": "fwd_pos", "mapped": "fwd_mapped", "join": "fwd_pos"}[variant]
        bwd = {"plain": "bwd", "pos": "bwd", "mapped": "bwd_mapped", "join": "bwd_join"}[variant]
        out |= {(fwd, nv, rows), (bwd, nv, rows)}
    out |= {("fwd_half", nv, rows) for nv, rows in E.LN_HALF_CASES}
    out |= {("bwd", nv, 0) for nv in E.LN_EMPTY_BWD}
    for rows, c in _params(D.test_layer_norm_fwd_bwd):
        out |= {("fwd", P.ln_instance(c), rows), ("bwd", P.ln_instance(c), rows)}
    for rows, c in _params(D.test_layer_norm_half_matches_fp32_upcast):
        out.add(("fwd_half", P.ln_instance(c), rows))
    for q, b, c, with_pos, _ in _params(S.test_layer_norm_branch_matches_the_unfused_graph):
        out |= {("fwd_pos" if with_pos else "fwd", P.ln_instance(c), q * b), ("bwd_join", P.ln_instance(c), q * b)}
    return out


def test_restated_rules_on_known_shapes():
    assert [P.ln_instance(c) for c in (128, 384, 1024, 64, 1152, 200)] == [1, 3, 8, None, None, None]
    assert P.ln_fwd_grid(165) == 21 and P.ln_bwd_blocks(165) == 3 and P.ln_bwd_last_block_rows(165) == 37
    assert P.ln_bwd_blocks(128) == 2 and P.ln_bwd_last_block_rows(128) == 64 and P.ln_bwd_blocks(0) == 0
    assert P.bn_slots(4) == 256 and P.bn_slots(1024) == 1 and P.bn_grid(16384, 512) == 528
    assert P.bn_strided(16384, 512) and not P.bn_strided(528, 1024) and P.bn_strided(529, 1024)
    assert not P.bn_channels_ok(12) and P.bn_channels_ok(4)
    assert P.stream_grid(1027 // 4 + 1) == 2 and not P.stream_strided(1027) and P.stream_strided(4 * 1056 * 256 + 4)
    assert not P.stream_strided(4 * 1056 * 256 + 3)
    assert P.norm_grid(3) == 1 and P.norm_grid(10 ** 7) == 528 and P.norm_strided(4 * 528 * 256 + 4)
    # FlatParameters starts every tensor on a 64-element boundary: no head, and only a tensor's end has a tail
    assert P.adamw_split(64, 16384) == (0, 4096, 0) and P.adamw_split(128, 1001) == (0, 250, 1)
    assert P.adamw_split(5, 2) == (2, 0, 0) and P.adamw_split(6, 9) == (2, 1, 3)
    # the step's matcher: 256 x 64 stages its cost; 1024 x 64 does not fit and reads global memory
    assert P.hungarian_staged(256, 64) and P.hungarian_staged(64, 256)
    assert P.hungarian_staged(1024, 64) is False and P.hungarian_staged(64, 1024) is False
    assert P.hungarian_scene(256, 64, 20) == (20, True) and P.hungarian_scene(16, 64, 70) == (64, False)
    assert P.hungarian_scene(256, 64, 0) == (0, None)


def test_dropout_twin_matches_hand_worked_values():
    # mix32(0) = 0; mix32(1) by hand from step_kernels.cu:20-25
    x = 1
    x ^= x >> 16; x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15; x = (x * 0x846CA68B) & 0xFFFFFFFF
    x ^= x >> 16
    assert int(P.mix32(0)) == 0 and int(P.mix32(1)) == x
    # the fp32 threshold: p * 2^32 is exact in fp32; p -> 1 saturates below 2^32
    assert P.drop_threshold(0.5) == 1 << 31 and P.drop_threshold(0.0) == 0
    assert P.drop_threshold(np.nextafter(np.float32(1), np.float32(0))) == 4294967040
    assert P.drop_threshold(0.1) == int(np.float32(0.1) * np.float32(2 ** 32))
    assert P.drop_scale(0.5) == np.float32(2.0)
    # one element by hand: seed 7, salt 3, index 2^32 + 5 (both halves of the index enter the hash)
    key = int(P.mix32((7 + 3 * 0x9E3779B1) & 0xFFFFFFFF))
    inner = int(P.mix32((5 * 0x85EBCA77 + 1 * 0xC2B2AE3D + 0x27D4EB2F) & 0xFFFFFFFF))
    h = int(P.mix32(key ^ inner))
    assert P.drop_keep(7, 3, 0.5, [(1 << 32) + 5])[0] == (h >= 1 << 31)
    assert P.drop_keep(7, 3, 0.0, [1, 2]).all()
    keep = P.drop_keep(12345, 678, 0.1, np.arange(1 << 20))
    assert abs(keep.mean() - 0.9) < 2e-3
    assert not np.array_equal(keep, P.drop_keep(12345 + 7919, 678, 0.1, np.arange(1 << 20)))


def test_layer_norm_cases_reach_every_instance_in_every_form():
    launches = _ln_launches()
    for form in ("fwd", "fwd_pos", "fwd_mapped", "fwd_half", "bwd", "bwd_mapped", "bwd_join"):
        assert {nv for f, nv, _ in launches if f == form} >= set(range(1, 9)), form
    fwd_rows = {rows for f, _, rows in launches if f.startswith("fwd")}
    assert any(0 < r < P.LN_WARPS for r in fwd_rows), "rows < 8"
    assert any(P.ln_fwd_grid(r) > 1 and r % P.LN_WARPS for r in fwd_rows), "ragged multi-block forward"
    for form in ("bwd", "bwd_mapped", "bwd_join"):
        for nv in range(1, 9):
            rows = {r for f, n, r in launches if f == form and n == nv}
            assert any(P.ln_bwd_blocks(r) > 1 and P.ln_bwd_last_block_rows(r) < P.LN_BWD_ROWS for r in rows), \
                (form, nv, "multi-block backward with a partial last block")
    assert {nv for f, nv, r in launches if f == "bwd" and r == 0} == set(range(1, 9)), "backward of no rows"


def test_bn_cases_reach_every_width_both_sides_of_the_grid_stride():
    seen = set()
    for c, rows, relu, p in E.BN_CASES:
        assert P.bn_channels_ok(c)
        seen.add((c, relu, p > 0, P.bn_strided(rows, c)))
        if not P.bn_strided(rows, c):
            assert P.bn_grid(rows, c) <= 3
    for c in P.BN_WIDTHS:
        for relu in (False, True):
            for drop in (False, True):
                for strided in (False, True):
                    assert (c, relu, drop, strided) in seen, (c, relu, drop, strided)
    assert {p for *_, p in E.BN_CASES if p > 0} == set(E.PS)


def test_dropout_cases_reach_every_tail_and_the_grid_stride():
    tails = {(P.scalar_tail(n), P.stream_strided(n)) for n, *_ in E.DROP_CASES}
    # every n % 4 on both sides of the grid stride (each case runs with and without a residual, and the backward)
    assert tails == {(t, s) for t in range(4) for s in (False, True)}
    assert {p for _, p, _, _ in E.DROP_CASES} == set(E.PS)
    assert len({seed for _, _, seed, _ in E.DROP_CASES}) >= 8
    assert any(seed >= 1 << 31 for _, _, seed, _ in E.DROP_CASES), "a seed with the top bit set"


def test_adamw_chunks_reach_every_head_tail_split():
    splits = [P.adamw_split(off, ln) for off, ln, _ in E.ADAMW_CHUNKS]
    assert {(h, t) for h, b, t in splits if b > 0} == {(h, t) for h in range(4) for t in range(4)}
    assert {ln for _, ln, _ in E.ADAMW_CHUNKS if ln < 4} == {1, 2, 3}
    assert any(b > P.THREADS for _, b, _ in splits), "a body the block loops over more than once"
    ends = sorted((off, off + ln) for off, ln, _ in E.ADAMW_CHUNKS)
    assert all(a[1] <= b[0] for a, b in zip(ends, ends[1:])), "chunks overlap"
    assert any(a[1] < b[0] for a, b in zip(ends, ends[1:])), "an inactive gap between chunks"
    assert any(a[1] == b[0] for a, b in zip(ends, ends[1:])), "a tensor split into several chunks"
    assert {wd for *_, wd in E.ADAMW_CHUNKS} >= {0.0, 0.05}
    assert ends[-1][1] < E.ADAMW_N
    runs = {(steps > 1, clip, gs != 1.0) for steps, clip, gs, _ in E.ADAMW_RUNS}
    assert runs == {(m, c, s) for m in (False, True) for c in ("off", "above", "below") for s in (False, True)}
    assert any(start >= 1000 for *_, start in E.ADAMW_RUNS)


def test_grad_norm_cases_reach_the_tail_and_the_grid_stride():
    ns = list(E.NORM_NS) + [E.ADAMW_N]
    assert {P.scalar_tail(n) for n in ns} == {0, 1, 2, 3}
    assert {P.scalar_tail(n) for n in ns if P.norm_strided(n)} == {0, 1, 2, 3}
    assert P.norm_strided(E.ADAMW_N) and P.scalar_tail(E.ADAMW_N)


def test_hungarian_cases_reach_both_layouts_and_orientations():
    seen = set()
    clamped = False
    for nprop, ngt, nact, ints in E.HUNG_CASES:
        if isinstance(nact, str):
            continue
        staged = P.hungarian_staged(nprop, ngt)
        assert staged is not None
        for a in nact:
            na, transposed = P.hungarian_scene(nprop, ngt, a)
            clamped |= a > ngt
            if na > 0:
                seen.add((staged, transposed, ints))
            else:
                seen.add((staged, None, ints))
    assert {(s, t) for s, t, _ in seen} >= {(s, t) for s in (False, True) for t in (False, True, None)}
    assert {t for s, t, i in seen if s is False and i and t is not None} == {False, True}, \
        "ties on the unstaged path in both orientations"
    assert clamped, "nactual > ngt"
    assert any(nact == "step" and (nprop, ngt) == (256, 64) for nprop, ngt, nact, _ in E.HUNG_CASES)


def test_remainder_cases():
    widths = {c for _, c in E.SOFTMAX_CASES}
    assert {1, 31, 32, 33} <= widths and max(widths) > 1024
    assert any(rows % 8 for rows, _ in E.SOFTMAX_CASES)
    assert any(count > 16 and alias is not None and alias >= 16 for _, count, alias in E.SUM_CASES)
    assert any(count > 32 and alias is not None and alias >= 32 for _, count, alias in E.SUM_CASES)
    assert {P.scalar_tail(n) for n, _, _ in E.SUM_CASES} >= {2, 3}
