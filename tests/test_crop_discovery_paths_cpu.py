"""The CLIP crop kernel's tap cap and its direct-form fallback never come into play, the ScanNet plan is what it is,
and the GPU tests of the crop kernel and of the novel-box candidate kernel reach every path and edge.

tests/crop_discovery_paths.py restates the rules of csrc/image_kernels.cu and csrc/discovery_kernels.cu; the proofs
enumerate every box edge and every tile of the shipped image sizes, and the coverage checks map the case lists of
test_clip_crop_edges_gpu.py and test_novel_candidates_edges_gpu.py through the rules.  Removing a case, or moving a
rule in the sources without a GPU case that runs the new side, fails here, without a GPU."""
import numpy as np
import pytest

import crop_discovery_paths as P
import test_clip_crop_edges_gpu as C
import test_novel_candidates_edges_gpu as N

SHIPPED = ((531, 730, 224), (530, 730, 224), (968, 1296, 224))     # SUN RGB-D (both heights), ScanNet, at CLIP's 224
SWEEP = tuple((m, m, res) for res in (16, 36, 64, 224, 336) for m in (res // 2, res, res + 1, 3 * res + 7))
SWEEP += ((2000, 2000, 224), (120, 160, 36), (170, 200, 160), (64, 96, 16), (1500, 900, 336))


def _plans(h, w, res):
    """every plan the kernel can run for an (h, w) image: the automatic one and tile_rows 1 ... 64"""
    plans = {P.crop_plan(h, w, res, t) for t in range(0, P.MAX_TILE_ROWS + 1)}
    assert None not in plans
    return plans


def _worst_margins(h, w, res):
    """-> (max over every box edge and filter of untruncated taps - cap, max over every tile of nsrc - rmax), under
    both readings of the span arithmetic (center rounded before the support is added, as compiled, or fused)"""
    plans = _plans(h, w, res)
    taps = {p.taps for p in plans}.pop()
    worst_taps = worst_src = -(1 << 30)
    for fused in (False, True):
        for edge in range(1, max(h, w) + 1):
            lo, n = P.aa_span(edge, res, fused)
            worst_taps = max(worst_taps, int(n.max()) - taps)
            for p in plans:
                worst_src = max(worst_src, int((P.tile_nsrc(lo, n, p.tr, p.taps) - p.rmax).max()))
    return worst_taps, worst_src


@pytest.mark.parametrize("h,w,res", SHIPPED + SWEEP)
def test_tap_cap_and_direct_form_never_fire(h, w, res):
    """aa_weights_to's `n = min(n, cap)` never drops a tap: a filter has at most cap - 1 taps (the cap is
    2 ceil(2 s) + 1 and a filter spans at most ceil(4 s) <= 2 ceil(2 s) source pixels); and every tile's source rows
    fit the shared buffer, so the direct form of image_kernels.cu:187-201 cannot run"""
    if P.crop_plan(h, w, res) is None:
        pytest.skip("refused by crop_plan")
    worst_taps, worst_src = _worst_margins(h, w, res)
    assert worst_taps <= -1, f"a filter reaches the tap cap ({worst_taps})"
    assert worst_src <= 0, f"a tile needs {worst_src} more source rows than the buffer holds"


def test_sweep_reaches_the_plans_it_should():
    assert all(P.crop_plan(h, w, res) is not None for h, w, res in SWEEP)
    assert P.crop_plan(2000, 2000, 224) == P.CropPlan(tr=2, rmax=57, taps=37, smem=188472)
    assert {P.crop_plan(h, w, res).tr for h, w, res in SWEEP} >= {16, 8, 2}


def test_scannet_plan_is_pinned():
    """968 x 1296 at 224: tile height 8, 25 taps, 223 968 B of the 225 280 B limit (a change to the carve-up shows
    here); SUN RGB-D: tile height 16, 15 taps"""
    assert P.crop_plan(968, 1296, 224) == P.CropPlan(tr=8, rmax=74, taps=25, smem=223968)
    assert P.CR_SMEM_LIMIT - 223968 == 1312
    assert P.crop_plan(531, 730, 224) == P.CropPlan(tr=16, rmax=70, taps=15, smem=204480)
    assert P.crop_plan(968, 1296, 224, tile_rows=64).tr == 8 and P.crop_plan(968, 1296, 224, tile_rows=5).tr == 5


def test_restated_rules_on_known_values():
    # scale 2 exactly: center 2 i + 1, support 4 -> lo = 2 i - 3 (clamped at 0), 8 taps inside the image
    lo, n = P.aa_span(448, 224)
    assert lo[:3].tolist() == [0, 0, 1] and n[2] == 8 and lo[100] == 197 and n[100] == 8 and lo[-1] + n[-1] == 448
    # upsampling: support 2 in source pixels
    lo, n = P.aa_span(1, 224)
    assert (lo == 0).all() and (n == 1).all()
    assert P.crop_geometry([10, 20, 15, 30]) == (5, 10, 10, 2, 0)
    assert P.hrow_branches([0, 0, 224, 224], 224) == {"inside"}
    assert P.hrow_branches([0, 0, 224, 100], 224) == {"inside", "white"}
    assert P.hrow_branches([0, 0, 100, 224], 224) == {"inside", "mixed"}
    assert P.crop_status(16, 16, 16, 65535) == "ok" and P.crop_status(16, 16, 16, 65536) == "einval"
    assert P.crop_status(16, 16, 16, 0) == "empty" and P.crop_status(16, 16, 16, 1, tile_rows=65) == "einval"
    assert P.crop_plan(200, 2400, 224) is None and P.crop_plan(16, 16, 2048) is None
    # the candidate kernel: q = 1024 needs 156 816 B, so MAXQ, not the 200 KiB cap, bounds q
    assert P.novel_candidates_smem(1024) == 156816
    assert max(P.novel_candidates_smem(q) for q in range(1, P.NC_MAXQ + 1)) <= P.NC_SMEM_CAP
    # every array at its type's alignment for every q (the float4 boxes at an offset of 4 q faulted for q % 4 != 0),
    # and inside the bytes the launcher asks for
    for q in range(1, P.NC_MAXQ + 1):
        lay = P.novel_candidates_layout(q)
        assert lay["box"] % 16 == 0 and all(lay[k] % 4 == 0 for k in ("score", "order", "sup", "keep")), q
        assert lay["ok"] + q <= P.novel_candidates_smem(q), q
    assert P.novel_candidates_status(1, 1024, 0, 1) == "ok" and P.novel_candidates_status(1, 1025, 0, 1) == "einval"
    assert P.novel_candidates_status(1, 1, 0, 0) == "einval" and P.novel_candidates_status(0, 5, 0, 1) == "empty"


def _crop_launches():
    """-> list of (shape name, plan, box, valid) of every crop the fp64 test checks, and the set of tile heights the
    bit-relation test runs"""
    out, trs = [], set()
    for name, (_, h, w, res) in C.SHAPES.items():
        scene, boxes, valid = C.crop_cases(name)
        plan = P.crop_plan(h, w, res)
        out += [(name, plan, boxes[i], bool(valid[i])) for i in range(len(boxes))]
        trs |= {plan.tr} | {P.crop_plan(h, w, res, t).tr for t in C.TILE_ROWS}
        assert scene.max() == C.SHAPES[name][0] - 1, f"{name}: no crop of the last image"
        assert (~valid).any(), f"{name}: no given-up crop"
    return out, trs


def test_crop_cases_reach_every_path():
    launches, trs = _crop_launches()
    assert {p.tr for _, p, _, _ in launches} >= {16, 8, 2}, "automatic tile heights"
    assert trs >= {1, 2, 4, 8, 16, 32, 64}, "explicit tile heights"
    assert any(P.crop_plan(h, w, res, 64).tr == 64 and res > 64 and res % 64
               for _, h, w, res in C.SHAPES.values()), "tile height 64 over several tiles, the last one partial"
    branches, regimes, full_filter, partial = set(), set(), False, False
    for name, plan, box, valid in launches:
        if not valid:
            continue
        res = C.SHAPES[name][3]
        wc, hc, edge, _, _ = P.crop_geometry(box)
        branches |= P.hrow_branches(box, res)
        regimes.add("up" if edge < res else "one" if edge == res else "down")
        lo, n = P.aa_span(edge, res)
        full_filter |= int(n.max()) == plan.taps - 1
        partial |= res % plan.tr != 0
        assert (P.tile_nsrc(lo, n, plan.tr, plan.taps) <= plan.rmax).all()
    assert branches == {"inside", "white", "mixed"}, branches
    assert regimes == {"up", "one", "down"}, regimes
    assert full_filter, "no filter with the most taps a box can have (cap - 1)"
    assert partial, "no partial last tile"
    boxes = [tuple(int(v) for v in b) for name, _, b, _ in launches]
    assert any(b[2] - b[0] == 1 and b[3] - b[1] == 1 for b in boxes), "1 x 1"
    assert any(b[2] - b[0] == 1 and b[3] - b[1] > 1 for b in boxes) and any(b[3] - b[1] == 1 and b[2] - b[0] > 1
                                                                          for b in boxes), "slivers"
    parities = {(max(b[2] - b[0], b[3] - b[1]) - min(b[2] - b[0], b[3] - b[1])) % 2 for b in boxes}
    assert parities == {0, 1}, "both centring parities"
    for name, (_, h, w, res) in C.SHAPES.items():
        mine = [tuple(int(v) for v in b) for n_, _, b, _ in launches if n_ == name]
        assert (0, 0, w, h) in mine, f"{name}: the whole image"
        assert any(b[2] == w for b in mine) and any(b[3] == h for b in mine), f"{name}: right and bottom border"
        if name != "large":
            edges = {max(b[2] - b[0], b[3] - b[1]) for b in mine}
            assert {res - 1, res, res + 1} <= edges, name


def test_crop_limits_are_run():
    nimg, h, w, res, n = C.MANY
    assert P.crop_status(h, w, res, n) == "ok" and n == P.MAX_CROPS
    assert P.crop_status(h, w, res, n + 1) == "einval"
    assert [P.crop_status(h, w, res, 1) for _, h, w, res in C.TOO_LARGE] == ["etoolarge"] * 2
    assert P.crop_plan(*C.TOO_LARGE[0][1:]) is None and P.crop_plan(*C.TOO_LARGE[1][1:]) is None


def test_candidate_cases_reach_every_edge():
    qs = set(N.QS)
    for edge in (32, 256):
        assert {edge - 1, edge, edge + 1} <= qs, edge
    assert P.NC_MAXQ in qs and all(P.novel_candidates_status(1, q, 0, 1) == "ok" for q in qs)
    assert any(P.novel_candidates_status(b, q, g, cap) == "einval" and q == P.NC_MAXQ + 1 for b, q, g, cap in N.REFUSED)
    assert any(P.novel_candidates_status(b, q, g, cap) == "einval" and cap == 0 for b, q, g, cap in N.REFUSED)
    assert 0 in N.GS and max(N.GS) == 64
    assert any(N.cap_of(c, q) > q for c in N.CAPS for q in N.QS), "cap > q"
    assert any(q > P.NC_THREADS for q in qs), "a block that loops over its boxes"
    assert N.MODEL_SHAPE == (8, 128, 64, 32)
    # cap < total: the oracle's untruncated count on the cases without ground truth, at the smallest capacity
    import discovery_ref
    truncated = False
    for q in (128, 1000):
        case = N.random_case(2, q, 0, seed=q * 7)
        _, cnt = discovery_ref.novel_candidates_ref(*case, *N.THRESHOLDS, q)
        truncated |= bool((cnt[:, 1] > min(N.cap_of(c, q) for c in N.CAPS)).any())
    assert truncated, "no case where the capacity truncates the list"


def test_normalisation_bound_holds_at_every_level():
    """the GPU test's bound on the normalised value, (ulp(u / 255) / 2 + ulp(u / 255 - mean) / 2) / std +
    ulp(result) / 2, holds for the kernel's fp32 steps at every channel and level, and a one-ulp change of the output
    breaks it.  In ulps of the value the error is not small: the difference cancels near the mean, so 2 ulps of the
    fp64 value cannot be required of any fp32 evaluation (170.6 ulps for channel 2 at level 104)."""
    u8 = np.broadcast_to(np.arange(256.0)[None, :, None], (3, 256, 1)).copy()
    o = C._normalised32(u8)
    err, bound, ulps = C.normalisation_error(o, u8)
    assert (err <= bound).all() and err.max() < 2.5e-7
    e2, b2, _ = C.normalisation_error(np.nextafter(o, np.float32(np.inf)), u8)
    assert (e2 > b2).any()
    assert np.unravel_index(ulps.argmax(), ulps.shape)[:2] == (2, 104) and 170 < ulps.max() < 171
    assert (ulps > 2).mean() > 0.1
