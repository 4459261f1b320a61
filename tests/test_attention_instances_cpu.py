"""The GPU tests of the wgmma attention kernels reach every instance in every variant, every tail and every ring wrap.

tests/attention_instances.py restates the launchers' instance selection, ring depths and tile walks; this maps the
case lists of test_attention_gpu.py and test_attention_edges_gpu.py through them.  Removing a case, or adding an
instance or moving a rule in csrc/ without a GPU case that runs it, fails here, without a GPU."""
import importlib.util
from pathlib import Path

import attention_instances as AI
import test_attention_edges_gpu as E
import test_attention_gpu as T

VARIANTS = set(E.VARIANTS)


def _bench_attention():
    path = Path(__file__).resolve().parents[1] / "tools" / "bench_attention.py"
    spec = importlib.util.spec_from_file_location("bench_attention", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _variant(masked: bool, p: float) -> str:
    return {(False, False): "plain", (True, False): "mask", (False, True): "dropout",
            (True, True): "mask+dropout"}[(masked, p > 0)]


def _forward_runs():
    """(lq, lk, hd, nsplit, variant) of every fp32-operand forward the GPU tests compare with fp64"""
    runs = [(lq, lk, hd, ns, "plain") for lq, lk, _, _, hd in T.CASES for ns, _ in T.NSPLIT_TOLS]
    runs += [(lq, lk, hd, 3, _variant(False, p)) for lq, lk, _, _, hd in T.BWD_CASES for p in (0.0, 0.1)]
    runs += [(lq, lk, hd, 3, _variant(True, p)) for lq, lk, _, _, hd in T.MASKED_CASES for p in (0.0, 0.1)]
    runs += list(E.FWD_CASES)
    runs += [(lq, 300, hd, ns, _variant(True, p)) for hd, lq in E.EDGE_CASES for p in (0.0, 0.1) for ns in (2, 3)]
    return runs


def _backward_runs():
    """(lq, lk, hd, variant) of every backward the GPU tests compare with fp64"""
    runs = [(lq, lk, hd, _variant(False, p)) for lq, lk, _, _, hd in T.BWD_CASES for p in (0.0, 0.1)]
    runs += [(lq, lk, hd, _variant(True, p)) for lq, lk, _, _, hd in T.MASKED_CASES for p in (0.0, 0.1)]
    runs += list(E.BWD_CASES)
    return runs


def test_restated_rules_on_known_shapes():
    # ring depths: 4 for every hd-64 forward but <64, 3, 2>; hd 128 by planes; backward 4 and 2
    assert {(ns, nwg): AI.fwd_nst(64, ns, nwg) for ns in (1, 2, 3) for nwg in (1, 2)} == {
        (1, 1): 4, (1, 2): 4, (2, 1): 4, (2, 2): 4, (3, 1): 4, (3, 2): 3}
    assert [AI.fwd_nst(128, ns, 1) for ns in (1, 2, 3)] == [4, 2, 1]
    assert AI.bwd_nst(64) == 4 and AI.bwd_nst(128) == 2
    assert len(AI.FWD_INSTANCES) == 10
    # the CLIP tower (50 tokens) runs one warpgroup; the encoder (2048) two; the decoder (hd 128) one
    assert AI.fwd_instance(50, 64, 2) == (64, 2, 1, False) and AI.fwd_instance(2048, 64, 2) == (64, 2, 2, False)
    assert AI.fwd_instance(2048, 128, 3) == (128, 3, 1, False)
    # the step's encoder walk: 32 key tiles of 4-stage rings, no tail
    w = AI.fwd_walk(2048, 2048, 64, 2)
    assert (w["key_tiles"], w["key_tail"], w["wraps"], w["q_tail_wg"]) == (32, False, 7, None)
    assert AI.fwd_walk(130, 200, 64, 3)["q_tail_wg"] == 0 and AI.fwd_walk(200, 200, 64, 3)["q_tail_wg"] == 1
    assert AI.wraps(256, 4) == 0 and AI.wraps(257, 4) == 1 and AI.wraps(513, 4) == 2
    bw = AI.bwd_walk(300, 37, 64)
    assert (bw["dq_tiles"], bw["dkv_tiles"], bw["lqp"], bw["k_tail_wg"]) == (1, 5, 320, 0)
    assert AI.half_out_accepted(50, 64, 2, False) and not AI.half_out_accepted(50, 64, 2, True)
    assert not AI.half_out_accepted(65, 64, 1, False) and not AI.half_out_accepted(50, 64, 3, False)
    assert AI.half_out_requested(50, 64, 2) and not AI.half_out_requested(50, 128, 2)


def test_forward_cases_reach_every_instance_variant_and_edge():
    runs = [(AI.fwd_walk(lq, lk, hd, ns), var) for lq, lk, hd, ns, var in _forward_runs()]
    fp32 = AI.FWD_INSTANCES - {(64, 1, 1, True)}
    for var in VARIANTS:
        assert {w["instance"] for w, v in runs if v == var} == fp32, var
    for inst in fp32:
        walks = [w for w, _ in runs if w["instance"] == inst]
        assert any(w["key_tiles"] == 1 for w in walks), inst
        assert any(w["key_tail"] for w in walks), inst
        assert any(w["wraps"] == 1 for w in walks), inst
        assert any(w["wraps"] >= 2 for w in walks), inst
        if inst[2] == 2:
            assert {w["q_tail_wg"] for w in walks} >= {0, 1}, inst
    # the fp16 instance of the CLIP tower, and fp16 output from every instance that has it (plain only)
    assert {AI.fwd_instance(l, 64, 1, f16=True) for l in E.HALF_CASES} == {(64, 1, 1, True)}
    assert {1, 64} <= set(E.HALF_CASES)
    half_out = {AI.fwd_instance(lq, 64, ns) for lq, lk, ns in E.HALF_OUT_CASES if AI.half_out_requested(lk, 64, ns)}
    assert half_out == {(64, ns, nwg, False) for ns in (1, 2) for nwg in (1, 2)}


def test_backward_cases_reach_every_instance_variant_and_edge():
    runs = [(AI.bwd_walk(lq, lk, hd), lq, lk, var) for lq, lk, hd, var in _backward_runs()]
    for var in VARIANTS:
        assert {w["instance"] for w, _, _, v in runs if v == var} == AI.BWD_INSTANCES, var
    for inst in AI.BWD_INSTANCES:
        mine = [(w, lq, lk) for w, lq, lk, _ in runs if w["instance"] == inst]
        assert any(w["dq_wraps"] >= 2 for w, _, _ in mine), inst
        assert any(w["dkv_wraps"] >= 2 for w, _, _ in mine), inst
        assert any(lq < 64 for _, lq, _ in mine) and any(lk < 64 for _, _, lk in mine), inst
        assert any(w["q_tail"] for w, _, _ in mine) and any(w["k_tail"] for w, _, _ in mine), inst
        assert any(w["lqp"] > lq for w, lq, _ in mine), inst        # padded rows of the (lse, D) array
        if inst[1] == 2:
            assert {w["q_tail_wg"] for w, _, _ in mine} >= {0, 1}, inst
            assert {w["k_tail_wg"] for w, _, _ in mine} >= {0, 1}, inst


def test_step_chain_runs_every_backward_shape_of_the_step():
    bench = {(b, h, lq, lk, hd, p) for _, b, h, lq, lk, hd, p, _ in _bench_attention().BWD_CASES}
    assert {(b, h, lq, lk, hd, E.P_DROP) for _, _, b, h, lq, lk, hd in E.CHAIN_CASES} == bench
    # the layouts of models/transformer.py: fused q|k|v (encoder), fused q|k + v (decoder self), three tensors (cross)
    assert {(c[0], c[1]) for c in E.CHAIN_CASES} == {
        ("encoder self", "qkv"), ("decoder self", "qk_v"), ("decoder cross", "q_k_v")}


def test_pattern_cases_read_out_every_instance_and_key_position():
    fwd = {(AI.fwd_instance(lq, hd, ns), var) for lq, lk, hd, ns, var in E.PATTERN_FWD_CASES}
    assert fwd == {(i, v) for i in AI.FWD_INSTANCES if not i[3] for v in E.PATTERN_VARIANTS}
    assert {AI.bwd_instance(hd) for hd, _ in E.PATTERN_BWD_CASES} == AI.BWD_INSTANCES
    assert {(hd, v) for hd, v in E.PATTERN_BWD_CASES} == {(hd, v) for hd in (64, 128) for v in E.PATTERN_VARIANTS}
    # key positions 0, 63, 64 and the last key of a partial tile, in every read-out
    shapes = list(E.PATTERN_FWD_SHAPES.values()) + list(E.PATTERN_DKV_SHAPES.values()) + \
        list(E.PATTERN_DQ_SHAPES.values())
    for lq, lk in shapes:
        assert lk > 64 and AI.tail(lk), (lq, lk)
    # the dK/dV read-out covers both warpgroups' key tiles and more than one query tile
    for hd, (lq, lk) in E.PATTERN_DKV_SHAPES.items():
        assert AI.tiles(lq) > 1 and (AI.bwd_nwg(hd) == 1 or lk > 64), hd
