"""The four evaluation kernels (include/coda_eval.h, csrc/eval_kernels.cu) one by one against the sequential fp64
references of oracle/box_ref64.py, at the sizes where their loops take one, two and many trips, on both sides of the
shared-memory opt-in, and on the inputs the golden evaluation set avoids on purpose: score ties, duplicate boxes, IoU
ties, boxes without volume, scores that are not numbers.  tests/test_eval_gpu.py covers the one shape of the golden
set end to end; inputs here are generated from seeds."""
import ctypes
import math

import numpy as np
import pytest
import torch

import box_ref64 as ref
from coda_neurips2023_b200._lib import CodaError, lib, ptr, stream_of
from coda_neurips2023_b200.utils import ap_calculator as apc
from coda_neurips2023_b200.utils.box_util import flip_axis_to_camera_tensor, get_3d_box_batch_tensor

pytestmark = pytest.mark.gpu

SIGNS = torch.tensor([[1, 1, 1], [1, 1, -1], [-1, 1, -1], [-1, 1, 1], [1, -1, 1], [1, -1, -1], [-1, -1, -1],
                      [-1, -1, 1]], dtype=torch.float32)


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


# --------------------------------------------------------------------------- nms3d
def _nms_scene(b, k, seed, tied_scores=True):
    """axis-aligned boxes crowded enough that most of them overlap a few others; a quarter of them exact duplicates
    of another quarter, a few without height; scores from five values, classes from three, ~85 % valid"""
    g = torch.Generator().manual_seed(seed)
    side = 0.9 * max(k, 2) ** (1 / 3)
    cen = torch.rand(b, k, 1, 3, generator=g) * side
    half = torch.rand(b, k, 1, 3, generator=g) * 0.4 + 0.2
    if k >= 8:
        cen[:, k // 4: 2 * (k // 4)] = cen[:, : k // 4]
        half[:, k // 4: 2 * (k // 4)] = half[:, : k // 4]
        half[:, -3:, :, 1] = 0.0                                 # zero volume
    corners = (cen + half * SIGNS).contiguous()
    if tied_scores:
        score = torch.randint(0, 5, (b, k), generator=g).float() * 0.2 + 0.1
    else:
        score = torch.rand(b, k, generator=g)
    cls = torch.randint(0, 3, (b, k), generator=g)
    valid = torch.rand(b, k, generator=g) < 0.85
    return corners, score, cls, valid


def _check_nms(corners, score, cls, valid, thresh, old_type):
    """keep == the sequential rule, scene by scene; a scene in which some decision sits within 1e-6 of the threshold
    (less than an fp32 overlap resolves) is left out and reported"""
    got = apc.nms3d(corners.cuda(), score.cuda(), valid.cuda(), thresh, None if cls is None else cls.cuda(),
                    bool(old_type)).cpu().numpy()
    skipped = 0
    for i in range(corners.shape[0]):
        exp, margin = ref.nms3d_ref(corners[i], score[i], None if cls is None else cls[i], valid[i], thresh, old_type)
        if margin < 1e-6:
            skipped += 1
            continue
        assert np.array_equal(got[i], exp), (i, int(got[i].sum()), int(exp.sum()))
    return skipped, got


NMS_CONFIGS = [(False, 0, 0.25), (True, 0, 0.25), (True, 1, 0.25), (False, 1, 0.25), (False, 0, 0.0), (True, 0, 0.0)]


@pytest.mark.parametrize("k", [1, 2, 255, 256, 257, 1000, 1199, 2048])
def test_nms3d_equals_sequential_rule(k):
    """one and several trips of the 256-thread loops, both sides of the 48 KiB shared-memory opt-in (k ~ 1198), the
    documented maximum; class-aware or not, both overlap definitions, thresholds 0.25 and 0; tied scores and duplicate
    boxes, where only the tie rule (higher index first) decides who survives"""
    b = 3 if k <= 1000 else 2
    skipped = scenes = 0
    for n, (use_cls, old, thr) in enumerate(NMS_CONFIGS):
        corners, score, cls, valid = _nms_scene(b, k, seed=1000 * n + k, tied_scores=(n % 2 == 0))
        s, got = _check_nms(corners, score, cls if use_cls else None, valid, thr, old)
        skipped += s
        scenes += b
        assert not got[~valid.numpy()].any()
        if k >= 255:
            assert 0 < got.sum() < valid.sum()                      # something is kept, something is suppressed
    assert skipped * 6 <= scenes, (skipped, scenes)


def test_nms3d_class_and_tie_rules_decide_on_a_hand_example():
    """the five boxes of tests/test_box_ref_cpu.py: cubes at x = 0, 0.5, 0.5 (duplicate), 3, and 0.25 of class 1"""
    cen = torch.tensor([0.0, 0.5, 0.5, 3.0, 0.25]).view(1, 5, 1, 1) * torch.tensor([1.0, 0.0, 0.0])
    corners = (cen + 0.5 * SIGNS).contiguous()
    score = torch.tensor([[0.9, 0.7, 0.7, 0.7, 0.8]])
    cls = torch.tensor([[0, 0, 0, 0, 1]])
    valid = torch.ones(1, 5, dtype=torch.bool)
    run = lambda thr, c=cls, old=False, v=valid: apc.nms3d(corners.cuda(), score.cuda(), v.cuda(), thr,
                                                           None if c is None else c.cuda(), old).cpu()[0].tolist()
    assert run(0.25) == [True, False, False, True, True]
    assert run(0.25, c=None) == [True, False, False, True, False]
    assert run(0.4) == [True, False, True, True, True]             # of the tied duplicates the higher index survives
    assert run(0.5, old=True) == [True, False, True, True, True]   # inter / vol_j = 0.5 exactly: strictly greater
    assert run(0.4, old=True) == [True, False, False, True, True]
    assert run(0.25, v=torch.tensor([[False, True, True, True, True]])) == [False, False, True, True, True]


def test_nms3d_validity_edges_and_size_limit():
    corners, score, cls, valid = _nms_scene(2, 300, seed=5)
    none = torch.zeros_like(valid)
    assert not apc.nms3d(corners.cuda(), score.cuda(), none.cuda(), 0.25, cls.cuda()).any()
    one = none.clone()
    one[0, 299] = one[1, 0] = True
    assert torch.equal(apc.nms3d(corners.cuda(), score.cuda(), one.cuda(), 0.25, None).cpu(), one)
    big = _nms_scene(1, 2049, seed=6)
    with pytest.raises(CodaError, match="nms3d"):
        apc.nms3d(big[0].cuda(), big[1].cuda(), big[3].cuda(), 0.25)


def test_nms3d_large_then_small_then_large():
    """the shared-memory opt-in is raised once per size: a small scene after a large one, and a large one again"""
    for k, seed in ((2048, 1), (8, 2), (1500, 3), (2048, 4), (1200, 5)):
        corners, score, cls, valid = _nms_scene(2, k, seed=seed)
        _check_nms(corners, score, cls, valid, 0.25, 0)


def test_nms3d_birds_eye_view_flattening():
    """select_detections' 2-D NMS: the same kernel on corners whose height is flattened to [0, 1]"""
    g = torch.Generator().manual_seed(9)
    k = 200
    size = torch.rand(2, k, 3, generator=g) * 1.0 + 0.3
    ang = (torch.rand(2, k, generator=g) * 2 - 1) * math.pi
    cen = torch.rand(2, k, 3, generator=g) * torch.tensor([5.0, 5.0, 1.0])
    flat = get_3d_box_batch_tensor(size, ang, flip_axis_to_camera_tensor(cen))
    flat[..., 1] = flat[..., 1] * 0 + (torch.arange(8) >= 4).float().view(1, 1, 8)
    score, valid = torch.rand(2, k, generator=g), torch.rand(2, k, generator=g) < 0.9
    skipped, got = _check_nms(flat, score, None, valid, 0.25, 0)
    assert skipped == 0 and 0 < got.sum() < valid.sum()


def test_nms3d_scores_that_are_not_ordinary_numbers():
    """-inf and +inf are scores like any other (a valid box scored -inf is still a candidate, visited last); a box
    whose score is NaN cannot be ranked and is not a candidate: never kept, and it suppresses nothing"""
    corners, score, cls, valid = _nms_scene(2, 300, seed=12)
    score[:, 10:40] = float("-inf")
    score[:, 40:45] = float("inf")
    score[:, 50:90] = float("nan")
    score[1, 0] = float("nan")
    valid[:, 10:20] = True
    skipped, got = _check_nms(corners, score, cls, valid, 0.25, 0)
    assert skipped == 0
    assert not got[torch.isnan(score).numpy()].any()
    assert got[:, 10:40].any() and got[:, 40:45].any()
    plain = torch.where(torch.isnan(score), torch.zeros_like(score), score)
    same = apc.nms3d(corners.cuda(), plain.cuda(), (valid & ~torch.isnan(score)).cuda(), 0.25, cls.cuda()).cpu().numpy()
    assert np.array_equal(got, same)


# --------------------------------------------------------------------------- points_in_boxes
def _rotated_boxes(b, k, seed):
    g = torch.Generator().manual_seed(seed)
    size = torch.rand(b, k, 3, generator=g) * 1.5 + 0.3
    ang = (torch.rand(b, k, generator=g) * 2 - 1) * math.pi
    cen = torch.rand(b, k, 3, generator=g) * torch.tensor([4.0, 4.0, 1.5])
    cen[:, 1::2, :2] += 10.0                                       # every other box 10 m out
    return get_3d_box_batch_tensor(size, ang, flip_axis_to_camera_tensor(cen)), cen


def _clear_points(corners, cen, n, seed):
    """n depth-frame fp32 points around the boxes of one scene, none within 1e-4 of an edge length of any face of
    any box (an fp32 dot product at 10 m resolves ~1e-6 of it)"""
    rng = np.random.default_rng(seed)
    k = corners.shape[0]
    out = np.zeros((0, 3), np.float32)
    while out.shape[0] < n:
        m = max(2 * (n - out.shape[0]), 64)
        p = (cen.numpy()[rng.integers(0, k, m)] + rng.uniform(-1.0, 1.0, (m, 3))).astype(np.float32)
        clear = np.ones(m, bool)
        for lo in range(0, k, 32):
            t = ref.points_in_boxes_coords(corners[lo:lo + 32], p)
            clear &= (np.minimum(np.abs(t), np.abs(t - 1)) > 1e-4).all(-1).all(0)
        out = np.concatenate((out, p[clear]))
    return out[:n]


@pytest.mark.parametrize("k,n,stride", [(1, 1025, 3), (127, 1023, 4), (128, 1024, 6), (129, 1, 3), (300, 1025, 4),
                                        (5, 20000, 6), (5, 0, 3), (130, 2049, 3)])
def test_points_in_boxes_equals_fp64_count(k, n, stride):
    """a second block of boxes whose dead lanes still take part in the barriers, point tiles of 1024 with and without
    a tail, no points at all; rows wider than three floats whose extra columns must not be read (they hold NaN)"""
    b = 2
    corners, cen = _rotated_boxes(b, k, seed=k + n)
    pts = torch.full((b, n, stride), float("nan"))
    for i in range(b):
        pts[i, :, :3] = torch.from_numpy(_clear_points(corners[i], cen[i], n, seed=i))
    got = apc.points_in_boxes(corners.cuda(), pts.cuda()).cpu().numpy()
    assert got.shape == (b, k) and got.dtype == np.int32
    exp = np.stack([ref.points_in_boxes_ref(corners[i], pts[i].numpy()) for i in range(b)])
    assert np.array_equal(got, exp)
    if n >= 1023:
        assert exp.sum() > 20


def test_points_in_boxes_faces_are_inclusive_and_flat_boxes_are_empty():
    """axis-aligned boxes and points on a grid of 2^-6 m, 10 m out: every product the kernel forms is exact, so a
    point ON a face, an edge or a corner counts and a point one grid step outside does not -- no tolerance involved.
    A box with an edge of length zero holds nothing, whatever lies in its plane."""
    q = 2.0 ** -6
    cen = torch.tensor([[10.0, 10.5, 0.25], [-3.0, 2.0, 1.0], [0.0, 0.0, 0.0], [10.0, 10.5, 0.25], [0.0, 0.0, 0.0]])
    size = torch.tensor([[64 * q, 32 * q, 16 * q], [2 * q, 2 * q, 2 * q], [128 * q, 128 * q, 128 * q],
                         [64 * q, 32 * q, 0.0], [0.0, 0.0, 0.0]])
    corners = get_3d_box_batch_tensor(size, torch.zeros(5), flip_axis_to_camera_tensor(cen))[None]
    assert (corners[0, 4] == 0).all()
    pts, inside = [], np.zeros(5, np.int64)
    for j in range(3):
        h = size[j] / 2
        for sx in (-1, 0, 1):
            for sy in (-1, 0, 1):
                for sz in (-1, 0, 1):
                    s = torch.tensor([sx, sy, sz], dtype=torch.float32)
                    pts.append(cen[j] + h * s)                         # centre, face centres, edge midpoints, corners
                    if (sx, sy, sz) != (0, 0, 0):
                        pts.append(cen[j] + (h + q) * s)               # one grid step beyond each of them
    pts = torch.stack(pts)[None].contiguous()
    exp = ref.points_in_boxes_ref(corners[0], pts[0].numpy())
    assert exp[:3].tolist()[:2] == [27, 27] and exp[2] >= 27 and exp[3] == 0 and exp[4] == 0
    got = apc.points_in_boxes(corners.cuda(), pts.cuda()).cpu().numpy()[0]
    assert np.array_equal(got, exp), (got, exp)
    # the all-zero box and the flat box among ordinary ones, in the second block of a 128-box grid row
    many, c = _rotated_boxes(1, 200, seed=3)
    many[0, 150] = 0.0
    many[0, 160, :, 1] = many[0, 160, 0, 1]
    p = torch.cat((torch.from_numpy(_clear_points(many[0, :150], c[0, :150], 3000, seed=1)), torch.zeros(50, 3)))[None]
    got = apc.points_in_boxes(many.cuda(), p.cuda()).cpu().numpy()[0]
    assert got[150] == 0 and got[160] == 0 and got[:150].sum() > 100


# --------------------------------------------------------------------------- box3d_iou: nothing to do
def test_box3d_iou_with_no_pairs_launches_nothing_and_an_odd_pair_count_is_complete():
    c = _rotated_boxes(2, 4, seed=1)[0].cuda()
    out = torch.full((64,), -7.0, device="cuda")
    i = lambda v: ctypes.c_int(v)
    for k1, k2 in ((0, 4), (4, 0), (0, 0)):
        assert lib().coda_box3d_iou(i(2), i(k1), i(k2), ptr(c), ptr(c), ptr(out), stream_of(c)) == 0
    assert lib().coda_box3d_iou(i(0), i(4), i(4), ptr(c), ptr(c), ptr(out), stream_of(c)) == 0
    torch.cuda.synchronize()
    assert (out == -7.0).all()
    assert apc.box3d_iou(c, c[:, :0]).shape == (2, 4, 0)
    # 43 x 3 = 129 pairs: one thread into a second block
    c1 = _rotated_boxes(2, 43, seed=2)[0]
    c2 = (c1[:, 40:43] + 0.05).contiguous()
    got = apc.box3d_iou(c1.cuda(), c2.cuda()).cpu().double().numpy()
    assert np.abs(got - ref.box3d_iou64(c1, c2)).max() < 3e-6 and (got[:, 42] > 0).any()


# --------------------------------------------------------------------------- eval_match
def _match_case(b, k, g, ncls, seed):
    """IoUs and scores from a handful of values: ties everywhere, IoUs exactly at the thresholds; scores of -inf
    and NaN (not a detection of the class); one scene without live detections, one without ground truth"""
    gen = torch.Generator().manual_seed(seed)
    iou = torch.tensor([0.0, 0.1, 0.25, 0.3, 0.5, 0.7])[torch.randint(0, 6, (b, k, g), generator=gen)]
    scores = torch.tensor([0.2, 0.4, 0.4, 0.6, 0.8, float("-inf"), float("nan")])[
        torch.randint(0, 7, (b, k, ncls), generator=gen)]
    det_mask = torch.rand(b, k, generator=gen) < 0.8
    gt_cls = torch.randint(0, min(ncls, 6), (b, g), generator=gen)
    gt_present = torch.rand(b, g, generator=gen) < 0.7
    det_mask[1] = False
    if b > 2:
        gt_present[2] = False
    return iou, scores, det_mask, gt_cls, gt_present


@pytest.mark.parametrize("ncls", [1, 3, 4, 5, 10, 200])
def test_eval_match_equals_sequential_rule(ncls):
    """whole and partial last blocks of four warps (one warp per class; 200 = ScanNet-200), detections and
    ground-truth boxes below, at and over a warp's 32 lanes, no ground truth at all"""
    true_pos = 0
    for k in (1, 31, 32, 33, 256):
        for g in (0, 1, 33, 64):
            if ncls == 200 and k == 256 and g not in (0, 64):
                continue
            case = _match_case(3, k, g, ncls, seed=k * 100 + g)
            for thr in (0.25, 0.5):
                got = apc.eval_match(*(t.cuda() for t in case), thr).cpu().numpy()
                exp = ref.eval_match_ref(*(t.numpy() for t in case), thr)
                assert got.shape == (3, ncls, k)
                assert np.array_equal(got, exp), (k, g, thr, int(got.sum()), int(exp.sum()))
                assert not got[1].any() and not got[2].any()
                true_pos += int(exp.sum())
    assert true_pos > 50


def test_eval_match_rules_on_a_hand_example():
    """the cases of tests/test_box_ref_cpu.py::test_eval_match_ref_rules on the device"""
    iou = torch.tensor([[[0.6, 0.6], [0.7, 0.1], [0.3, 0.5]]])
    gt_cls, present = torch.tensor([[0, 0]]), torch.tensor([[True, True]])
    dm = torch.ones(1, 3, dtype=torch.bool)
    run = lambda sc, thr=0.25, m=dm: apc.eval_match(iou.cuda(), torch.tensor(sc).view(1, 3, 1).cuda(), m.cuda(),
                                                    gt_cls.cuda(), present.cuda(), thr).cpu()[0, 0].tolist()
    assert run([0.9, 0.8, 0.7]) == [True, False, True]      # first of two equal maxima; 1 finds its box claimed
    assert run([0.5, 0.5, 0.5]) == [True, False, True]      # equal scores: lower index first
    assert run([0.1, 0.8, 0.7]) == [False, True, True]      # 0's first maximum is claimed: no second choice
    assert run([0.9, 0.8, 0.7], thr=0.5) == [True, False, False]   # 2: IoU 0.5 is not greater than 0.5
    assert run([0.9, float("-inf"), float("nan")]) == [True, False, False]
    assert run([0.9, 0.8, 0.7], m=torch.tensor([[False, True, True]])) == [False, True, True]
