"""The fp64 box references of oracle/box_ref64.py, checked on the host before any kernel is compared with them:
the polygon intersection against an independent construction (scipy half-space intersection + convex hull), closed
forms, invariances of the reference itself, the NMS rule on a hand-worked example, and the edge-frame point test
against the reference project's own definition (a Delaunay hull test on the depth-frame corners)."""
import numpy as np
import pytest
import torch

import box_ref64 as ref
from coda_neurips2023_b200.utils.box_util import flip_axis_to_camera_tensor, get_3d_box_batch_tensor


def _rect(cx, cy, w, h, ang):
    c, s = np.cos(ang), np.sin(ang)
    pts = np.array([[-w, -h], [w, -h], [w, h], [-w, h]]) * 0.5
    return pts @ np.array([[c, s], [-s, c]]) + np.array([cx, cy])


def _halfspace_area(r1, r2):
    """Intersection area of two convex counter-clockwise quadrilaterals without any clipping: the Chebyshev centre
    of the eight half-planes (a linear programme) gives an interior point or shows there is none, then
    scipy.spatial.HalfspaceIntersection lists the vertices and ConvexHull measures them."""
    from scipy.optimize import linprog
    from scipy.spatial import ConvexHull, HalfspaceIntersection

    hs = []
    for r in (r1, r2):
        for i in range(4):
            a, b = r[i - 1], r[i]
            n = np.array([b[1] - a[1], a[0] - b[0]])          # outward normal of a counter-clockwise polygon
            n = n / np.linalg.norm(n)
            hs.append([n[0], n[1], -n @ a])                   # n.x + off <= 0
    hs = np.array(hs)
    res = linprog([0, 0, -1], A_ub=np.hstack((hs[:, :2], np.ones((8, 1)))), b_ub=-hs[:, 2],
                  bounds=[(None, None), (None, None), (0, None)])
    if not res.success or res.x[2] < 1e-9:
        return 0.0
    return ConvexHull(HalfspaceIntersection(hs, res.x[:2]).intersections).volume


def test_clip_area64_equals_halfspace_intersection():
    rng = np.random.default_rng(0)
    checked = overlapping = 0
    for t in range(60):
        far = rng.choice([0.0, 10.0])
        r1 = _rect(far + rng.uniform(-1, 1), far + rng.uniform(-1, 1), rng.uniform(0.2, 2), rng.uniform(0.2, 2),
                   rng.uniform(-np.pi, np.pi))
        r2 = _rect(far + rng.uniform(-1, 1), far + rng.uniform(-1, 1), rng.uniform(0.2, 2), rng.uniform(0.2, 2),
                   rng.uniform(-np.pi, np.pi))
        exp = _halfspace_area(r1, r2)
        got = ref.clip_area64(r1, r2)
        assert abs(got - exp) < 1e-9 * max(1.0, exp), (t, got, exp)
        # either winding of either polygon, and either of them as the subject
        assert abs(ref.clip_area64(r2[::-1], r1[::-1]) - exp) < 1e-9 * max(1.0, exp)
        checked += 1
        overlapping += exp > 1e-3
    assert checked == 60 and 20 < overlapping < 60


def test_clip_area64_closed_forms():
    unit = _rect(0, 0, 2, 2, 0)
    # a square of diagonal 2 turned by 45 degrees inside the square of side 2: its own area, 2
    assert abs(ref.clip_area64(_rect(0, 0, np.sqrt(2), np.sqrt(2), np.pi / 4), unit) - 2.0) < 1e-12
    # a square of side 2 turned by 45 degrees over the square of side 2: the regular octagon, 8 (sqrt 2 - 1)
    assert abs(ref.clip_area64(_rect(0, 0, 2, 2, np.pi / 4), unit) - 8 * (np.sqrt(2) - 1)) < 1e-12
    assert abs(ref.clip_area64(_rect(0.5, 0.25, 2, 2, 0), unit) - 1.5 * 1.75) < 1e-12
    assert ref.clip_area64(_rect(0.1, -0.2, 0.5, 0.3, 0.7), unit) == pytest.approx(0.15, abs=1e-12)   # contained
    assert ref.clip_area64(_rect(5, 0, 2, 2, 0.3), unit) == 0.0                                       # disjoint
    assert ref.clip_area64(_rect(2, 0, 2, 2, 0), unit) == 0.0                                         # sharing an edge
    assert ref.clip_area64(unit, np.zeros((4, 2))) == 0.0                                             # no interior


def _boxes(size, ang, cen):
    t = lambda a: torch.tensor(a, dtype=torch.float64)
    return get_3d_box_batch_tensor(t(size), t(ang), flip_axis_to_camera_tensor(t(cen)))[None]


def test_iou_and_giou_closed_forms():
    a = _boxes([[1.0, 2.0, 0.5]], [0.0], [[0.3, 0.2, 0.1]])
    one = torch.tensor([1])
    assert ref.box3d_iou64(a, a)[0, 0, 0] == pytest.approx(1.0, abs=1e-12)
    for rot in (False, True):
        assert ref.giou3d64(a, a, one, rot)[0, 0, 0] == pytest.approx(1.0, abs=1e-12)
    # disjoint along x: IoU 0, GIoU = -(1 - union / enclosing) with union = 2 and enclosing = 4 x 2 x 0.5
    far = _boxes([[1.0, 2.0, 0.5]], [0.0], [[3.3, 0.2, 0.1]])
    assert ref.box3d_iou64(a, far)[0, 0, 0] == 0.0
    for rot in (False, True):
        assert ref.giou3d64(a, far, one, rot)[0, 0, 0] == pytest.approx(-(1 - 2.0 / 4.0), abs=1e-12)
    # a box inside another: IoU = GIoU = small volume / large volume (the enclosing box is the large one)
    small = _boxes([[0.5, 0.5, 0.25]], [0.4], [[0.3, 0.2, 0.1]])
    assert ref.box3d_iou64(small, a)[0, 0, 0] == pytest.approx(0.0625, abs=1e-12)
    assert ref.giou3d64(small, a, one, True)[0, 0, 0] == pytest.approx(0.0625 - (1 - 1.0 / 1.0), abs=1e-12)
    # half overlap along the height only
    up = _boxes([[1.0, 2.0, 0.5]], [0.0], [[0.3, 0.2, 0.35]])
    assert ref.box3d_iou64(a, up)[0, 0, 0] == pytest.approx(0.5 / 1.5, abs=1e-12)
    # masked column, and the column rule of the rotated path: no intersection, the enclosing term stays
    two = torch.cat((a, a), dim=1)
    g = ref.giou3d64(a, two, torch.tensor([1]), True)
    assert g[0, 0, 1] == 0.0
    g = ref.giou3d64(a, two, torch.tensor([2]), True, rot_k2_limit=1)
    assert g[0, 0, 0] == pytest.approx(1.0, abs=1e-12) and g[0, 0, 1] == pytest.approx(-(1 - 2.0 / 1.0), abs=1e-12)
    # a box without extent is not `good`
    zero = torch.zeros(1, 1, 8, 3, dtype=torch.float64)
    assert ref.giou3d64(zero, zero, one, True)[0, 0, 0] == 0.0 and ref.box3d_iou64(zero, a)[0, 0, 0] == 0.0


def test_reference_is_translation_and_quarter_turn_invariant():
    rng = np.random.default_rng(1)
    n = 40
    size = rng.uniform(0.2, 2.0, (2, n, 3))
    ang = rng.uniform(-np.pi, np.pi, (2, n))
    cen = rng.uniform(-1.0, 1.0, (2, n, 3))
    c1, c2 = _boxes(size[0], ang[0], cen[0]), _boxes(size[1], ang[1], cen[1])
    nk = torch.tensor([n])
    iou, giou = ref.box3d_iou64(c1, c2), ref.giou3d64(c1, c2, nk, True)
    assert (iou > 0.05).sum() > 50
    shift = torch.tensor([8.0, -3.0, 16.0], dtype=torch.float64)
    assert np.abs(ref.box3d_iou64(c1 + shift, c2 + shift) - iou).max() < 1e-12
    assert np.abs(ref.giou3d64(c1 + shift, c2 + shift, nk, True) - giou).max() < 1e-12
    # a quarter turn of the scene about the up axis, (x, z) -> (z, -x): the IoU is a property of the pair.  (The
    # GIoU's enclosing box is axis-aligned and its `non_rot` gate reads two fixed corners, so it is not.)
    turn = lambda c: torch.stack((c[..., 2], c[..., 1], -c[..., 0]), dim=-1)
    assert np.abs(ref.box3d_iou64(turn(c1), turn(c2)) - iou).max() < 1e-12


def test_nms3d_ref_hand_worked_example():
    """Five boxes on a line: unit cubes at x = 0, 0.5 (IoU 1/3 with the first), 0.5 again (a duplicate), 3 and a
    cube at 0.25 of another class.  Scores 0.9, 0.7, 0.7, 0.7, 0.8."""
    def cube(x):
        return _boxes([[1.0, 1.0, 1.0]], [0.0], [[x, 0.0, 0.0]])[0, 0]
    corners = torch.stack([cube(0.0), cube(0.5), cube(0.5), cube(3.0), cube(0.25)])
    score = np.array([0.9, 0.7, 0.7, 0.7, 0.8])
    cls = np.array([0, 0, 0, 0, 1])
    valid = np.ones(5, bool)
    # visit order 0, 4, then the three tied boxes from the higher index: 3, 2, 1
    keep, margin = ref.nms3d_ref(corners, score, cls, valid, 0.25)
    assert keep.tolist() == [True, False, False, True, True]        # 0 drops 1 and 2 (1/3 > 0.25); 4 is another class
    assert margin == pytest.approx(1 / 3 - 0.25)
    keep, _ = ref.nms3d_ref(corners, score, None, valid, 0.25)
    assert keep.tolist() == [True, False, False, True, False]       # class-agnostic: 0 drops 4 too (IoU 0.6)
    keep, _ = ref.nms3d_ref(corners, score, cls, valid, 0.4)
    assert keep.tolist() == [True, False, True, True, True]         # 1/3 <= 0.4: of the duplicates index 2 goes first
    keep, _ = ref.nms3d_ref(corners, score, cls, valid, 1 / 3)
    assert keep.tolist() == [True, False, True, True, True]         # strictly greater than the threshold
    keep, _ = ref.nms3d_ref(corners, score, cls, np.array([0, 1, 1, 1, 1], bool), 0.25)
    assert keep.tolist() == [False, False, True, True, True]
    keep, _ = ref.nms3d_ref(corners, np.array([0.9, np.nan, 0.7, -np.inf, 0.8]), cls, valid, 0.4)
    assert keep.tolist() == [True, False, True, True, True]         # NaN: no candidate; -inf: an ordinary score
    # old type: intersection over the LATER box's volume -- 0.5 for the pair (0, 1)
    keep, _ = ref.nms3d_ref(corners, score, cls, valid, 0.4, old_type=True)
    assert keep.tolist() == [True, False, False, True, True]
    # zero volume: 0 / 0 is not greater than anything
    flat = corners.clone()
    flat[1, :, 1] = 0.0
    flat[2, :, 1] = 0.0
    keep, _ = ref.nms3d_ref(flat, score, cls, valid, 0.0, old_type=True)
    assert keep.tolist() == [True, True, True, True, True]


def test_points_in_boxes_ref_equals_delaunay_hull_test():
    """The reference project decides `inside` with scipy Delaunay(depth-frame corners).find_simplex(p) >= 0; the
    edge-frame rule is the same set except within rounding of a face."""
    from scipy.spatial import Delaunay

    rng = np.random.default_rng(2)
    k, n = 12, 4000
    size = rng.uniform(0.3, 2.0, (k, 3))
    ang = rng.uniform(-np.pi, np.pi, k)
    cen = rng.uniform(-1.0, 1.0, (k, 3)) + np.array([10.0, 0.0, 0.0]) * (np.arange(k)[:, None] % 2)
    corners = _boxes(size, ang, cen)[0].float()
    pts = (cen[rng.integers(0, k, n)] + rng.uniform(-1.2, 1.2, (n, 3))).astype(np.float32)
    t = ref.points_in_boxes_coords(corners, pts)
    counts = ref.points_in_boxes_ref(corners, pts)
    cam = corners.double().numpy()
    depth = np.stack((cam[..., 0], cam[..., 2], -cam[..., 1]), axis=-1)
    total = 0
    for j in range(k):
        hull = Delaunay(depth[j]).find_simplex(pts.astype(np.float64)) >= 0
        mine = ((t[j] >= 0) & (t[j] <= 1)).all(-1)
        clear = (np.minimum(np.abs(t[j]), np.abs(t[j] - 1)) > 1e-5).all(-1)
        assert np.array_equal(hull[clear], mine[clear]), j
        assert clear.mean() > 0.99 and mine.sum() == counts[j]
        total += int(mine.sum())
    assert total > 300
    # faces are inclusive, an edge of length zero leaves no inside
    cube = _boxes([[2.0, 2.0, 2.0]], [0.0], [[0.0, 0.0, 0.0]])[0]
    on = np.array([[1.0, 0.0, 0.0], [1.0, 1.0, 1.0], [-1.0, 1.0, 0.5], [0.0, 0.0, 0.0], [1.0 + 1e-9, 0.0, 0.0]])
    assert ref.points_in_boxes_ref(cube, on).tolist() == [4]
    flat = cube.clone()
    flat[:, :, 1] = 0.0
    assert ref.points_in_boxes_ref(flat, on).tolist() == [0]
    assert ref.points_in_boxes_ref(torch.zeros(1, 8, 3), np.zeros((3, 3))).tolist() == [0]


def test_eval_match_ref_rules():
    # one scene, one class, three detections, two ground-truth boxes
    iou = np.array([[[0.6, 0.6], [0.7, 0.1], [0.3, 0.5]]])
    gt_cls, present = np.array([[0, 0]]), np.array([[1, 1]])
    dm = np.ones((1, 3), bool)
    run = lambda sc, thr=0.25, m=dm: ref.eval_match_ref(iou, np.array(sc, dtype=np.float32).reshape(1, 3, 1), m, gt_cls,
                                                        present, thr)[0, 0].tolist()
    assert run([0.9, 0.8, 0.7]) == [True, False, True]   # 0 takes the first of its two equal maxima; 1 wants it too
    assert run([0.5, 0.5, 0.5]) == [True, False, True]   # equal scores: by ascending index
    # 1 claims box 0, 2 claims box 1; 0 then looks up its first maximum (box 0, claimed) and is a false positive: it
    # does not fall through to another box
    assert run([0.1, 0.8, 0.7]) == [False, True, True]
    assert run([0.9, 0.8, 0.7], thr=0.6) == [False, True, False]          # strictly greater than the threshold
    assert run([0.9, -np.inf, np.nan]) == [True, False, False]            # no detections of this class
    assert run([0.9, 0.8, 0.7], m=np.array([[0, 1, 1]], bool)) == [False, True, True]
    assert not ref.eval_match_ref(iou, np.ones((1, 3, 2), np.float32), dm, gt_cls, present, 0.25)[0, 1].any()
