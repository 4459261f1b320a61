"""coda_giou3d (matcher cost, csrc/detr_kernels.cu) and coda_box3d_iou (evaluation, csrc/eval_kernels.cu) against the
fp64 references of oracle/box_ref64.py, which are written from the definitions and checked on the host by
tests/test_box_ref_cpu.py -- unlike oracle/giou_ref.py, which restates the kernel's own fp32 arithmetic and so
cannot see an error both sides share.

What is varied is what the polygon clip is sensitive to: how far from the origin the pair stands (the clip works on
coordinates relative to one of its corners, so this must not matter), how small the boxes are, rotated or not, and
how the pair overlaps; then the edges of the index space and the degenerate boxes with a defined result."""
import math

import numpy as np
import pytest
import torch

import box_ref64 as ref
from coda_neurips2023_b200 import ops
from coda_neurips2023_b200.utils import ap_calculator as apc
from coda_neurips2023_b200.utils.box_util import flip_axis_to_camera_tensor, get_3d_box_batch_tensor

pytestmark = pytest.mark.gpu

OFFSETS = (0.0, 2.5, 5.0, 10.0, 20.0)
# |IoU - fp64| and |GIoU - fp64|.  The clip sees coordinates relative to a corner of the pair, a few box edges s at
# most for pairs that can intersect.  A crossing point is a quotient of differences of products of two such
# coordinates, each product rounded to 2^-24 of itself, so a crossing is off by a few 2^-24 s (more where two edges
# cross at a flat angle and the divisor is small) and the intersection area by a few 2^-24 s^2 per crossing, against a
# union of the order of s^2: some 1e-6 for the up to eight crossings together with the 2^-24 relative steps of the
# volumes, the union and the quotient -- at every scale and, because the coordinates are relative, at every distance.
# 3e-6 is that with room for a flat crossing; the worst pair of these sets measures 6.1e-7 (H100 80GB HBM3, 700 W).
ATOL = 3e-6


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def _pair_sets(scale, rotated, seed, offset=(0.0, 0.0, 0.0), b=2, k1=24, k2=12):
    """fp32 corners c1 (b, k1, 8, 3), c2 (b, k2, 8, 3) of boxes with edges of 0.4 .. 1.6 x scale in a cluster a few
    boxes wide around `offset` (depth frame: x, y horizontal, z up).  Of c2, per scene: three near copies of boxes of
    c1 (heavy overlap), three boxes inside boxes of c1, three that reach only into a corner region of one, the rest
    anywhere in the cluster (many disjoint from most of c1).  The same seed gives the same shapes at every offset."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    size1, size2 = (rnd(b, k1, 3) * 1.2 + 0.4) * scale, (rnd(b, k2, 3) * 1.2 + 0.4) * scale
    ang1 = (rnd(b, k1) * 2 - 1) * math.pi if rotated else torch.zeros(b, k1, dtype=torch.float64)
    ang2 = (rnd(b, k2) * 2 - 1) * math.pi if rotated else torch.zeros(b, k2, dtype=torch.float64)
    cen1 = (rnd(b, k1, 3) * 2 - 1) * torch.tensor([3.0, 3.0, 1.0]) * scale
    cen2 = (rnd(b, k2, 3) * 2 - 1) * torch.tensor([3.0, 3.0, 1.0]) * scale
    cen2[:, 0:3] = cen1[:, 0:3] + (rnd(b, 3, 3) - 0.5) * 0.2 * scale
    size2[:, 0:3] = size1[:, 0:3] * (0.9 + 0.2 * rnd(b, 3, 3))
    ang2[:, 0:3] = ang1[:, 0:3] + (0.3 * (rnd(b, 3) - 0.5) if rotated else 0.0)
    cen2[:, 3:6] = cen1[:, 3:6] + (rnd(b, 3, 3) - 0.5) * 0.1 * scale
    size2[:, 3:6] = size1[:, 3:6] * 0.3
    # towards a corner of the c1 box: along its own diagonal in the ground plane, by 0.9 of both half diagonals
    diag = 0.45 * (size1[:, 6:9, :2].norm(dim=-1) + size2[:, 6:9, :2].norm(dim=-1))
    phi = -ang1[:, 6:9] + torch.atan2(size1[:, 6:9, 1], size1[:, 6:9, 0])
    cen2[:, 6:9, 0] = cen1[:, 6:9, 0] + diag * torch.cos(phi)
    cen2[:, 6:9, 1] = cen1[:, 6:9, 1] + diag * torch.sin(phi)
    cen2[:, 6:9, 2] = cen1[:, 6:9, 2]
    off = torch.tensor(offset, dtype=torch.float64)
    mk = lambda s, a, c: get_3d_box_batch_tensor(s.float(), a.float(), flip_axis_to_camera_tensor((c + off).float()))
    return mk(size1, ang1, cen1), mk(size2, ang2, cen2)


def _errors(c1, c2, rotated):
    """worst |kernel - fp64| of the IoU (rotated clip always) and of the GIoU, plus the fp64 IoU for the mix checks"""
    nk = torch.full((c1.shape[0],), c2.shape[1], dtype=torch.int32)
    iou = apc.box3d_iou(c1.cuda(), c2.cuda()).cpu().double().numpy()
    giou = ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), rotated).cpu().double().numpy()
    iou64, giou64 = ref.box3d_iou64(c1, c2), ref.giou3d64(c1, c2, nk, rotated)
    return np.abs(iou - iou64).max(), np.abs(giou - giou64).max(), iou64


@pytest.mark.parametrize("rotated", [True, False], ids=["rotated", "axis_aligned"])
@pytest.mark.parametrize("scale", [0.05, 0.3, 1.5])
def test_iou_giou_vs_fp64_at_every_distance_from_the_origin(scale, rotated):
    """The same 576 pairs, moved 0 .. 20 m from the origin along x and z (depth x and y): the error against fp64 stays
    within ATOL in every cell, and at 20 m it is what it is at the origin (within 4x: the coordinates are rounded to a
    coarser grid out there, the arithmetic on them is the same)."""
    worst = {}
    for off in OFFSETS:
        c1, c2 = _pair_sets(scale, rotated, seed=int(scale * 100), offset=(off, off, 0.0))
        e_iou, e_giou, iou64 = _errors(c1, c2, rotated)
        worst[off] = (e_iou, e_giou)
        print(f"BOXGEOM scale {scale} m {'rotated' if rotated else 'axis-aligned'} offset {off:4.1f} m: "
              f"max |IoU - fp64| {e_iou:.2e}  max |GIoU - fp64| {e_giou:.2e}")
        # the mix: heavy overlap, containment, slight overlap, and a majority of disjoint pairs
        assert (iou64 > 0.5).sum() >= 4 and ((iou64 > 0) & (iou64 < 0.05)).sum() >= 4 and (iou64 == 0).mean() > 0.3
    bad = {off: e for off, e in worst.items() if not max(e) < ATOL}
    assert not bad, bad
    for q in (0, 1):
        assert worst[20.0][q] <= 4 * worst[0.0][q] + 2 ** -22, (q, worst)


@pytest.mark.parametrize("scale", [0.05, 1.5])
def test_iou_giou_vs_fp64_offset_along_the_up_axis(scale):
    c1, c2 = _pair_sets(scale, True, seed=7, offset=(0.0, 0.0, 20.0))
    e_iou, e_giou, _ = _errors(c1, c2, True)
    print(f"BOXGEOM scale {scale} m rotated, 20 m up: max |IoU - fp64| {e_iou:.2e}  max |GIoU - fp64| {e_giou:.2e}")
    assert e_iou < ATOL and e_giou < ATOL


@pytest.mark.parametrize("scale", [0.05, 0.3, 1.5])
def test_translation_by_a_power_of_two_changes_no_bit(scale):
    """Corners snapped to a grid of 2^-14 m and the pair moved by (8, 16, 8) m: every coordinate of both copies is an
    fp32 number, so every difference either kernel forms -- the clip's re-centring, heights, edges, extents -- is the
    same number in both copies, and IoU and GIoU must be EQUAL, not close.  (Exact by construction; for coordinates
    that are not on such a grid only the ATOL bound above is claimed.)"""
    c1, c2 = _pair_sets(scale, True, seed=11)
    grid = 2.0 ** -14
    c1, c2 = torch.round(c1 / grid) * grid, torch.round(c2 / grid) * grid
    assert float(c1.abs().max()) < 8 and float(c2.abs().max()) < 8       # (8 + 16) / 2^-14 steps: far below 2^24
    shift = torch.tensor([8.0, 16.0, 8.0])
    s1, s2 = c1 + shift, c2 + shift
    assert torch.equal(s1.double(), c1.double() + shift.double()) and torch.equal(s2.double(), c2.double() + shift.double())
    nk = torch.full((c1.shape[0],), c2.shape[1], dtype=torch.int32).cuda()
    iou, iou_s = apc.box3d_iou(c1.cuda(), c2.cuda()), apc.box3d_iou(s1.cuda(), s2.cuda())
    g, g_s = ops.giou3d(c1.cuda(), c2.cuda(), nk, True), ops.giou3d(s1.cuda(), s2.cuda(), nk, True)
    assert int((iou > 0).sum()) > 20
    assert torch.equal(iou, iou_s)
    assert torch.equal(g, g_s)
    assert np.abs(iou.cpu().double().numpy() - ref.box3d_iou64(c1, c2)).max() < ATOL


@pytest.mark.parametrize("b,k1,k2", [(1, 5, 1), (33, 7, 5), (2, 43, 3), (1, 1, 12), (3, 16, 8)])
def test_giou3d_index_space_edges(b, k1, k2):
    """k1 * k2 below, at and just over a multiple of the 128-thread block, one column, many scenes; nums_k2 of 0, k2
    and in between (masked columns exactly 0); the rotated clip limited to the first 4 columns or to all; the flag
    given on the host or read from the device."""
    c1, c2 = _pair_sets(0.5, True, seed=b * 100 + k1, offset=(5.0, 5.0, 0.0), b=b, k1=max(k1, 9), k2=max(k2, 9))
    c1, c2 = c1[:, :k1].contiguous(), c2[:, :k2].contiguous()
    nk = torch.tensor([(0, k2, k2 // 2, 1)[i % 4] for i in range(b)], dtype=torch.int32)
    if b == 1:
        nk[0] = k2
    for rotated in (True, False):
        for limit in (None, 4, k2):
            got = ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), rotated, limit)
            exp = ref.giou3d64(c1, c2, nk, rotated, limit)
            assert np.abs(got.cpu().double().numpy() - exp).max() < ATOL, (rotated, limit)
            for i in range(b):
                assert (got[i, :, int(nk[i]):] == 0).all()
            flag = torch.tensor([1 if rotated else 0], device="cuda", dtype=torch.int32)
            assert torch.equal(ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), flag, limit), got)
    iou = apc.box3d_iou(c1.cuda(), c2.cuda()).cpu().double().numpy()
    assert np.abs(iou - ref.box3d_iou64(c1, c2)).max() < ATOL


def test_giou3d_columns_beyond_the_rotated_limit_keep_the_enclosing_term():
    """rot_k2_limit = 4 (what the reference's compiled clip does): from column 4 on the intersection is 0 although the
    boxes overlap, and the GIoU is -(1 - (vol1 + vol2) / enclosing), not 0 and not what the full clip gives."""
    c1, c2 = _pair_sets(0.5, True, seed=5)
    nk = torch.full((2,), 12, dtype=torch.int32)
    full = ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), True, 12).cpu().double().numpy()
    lim = ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), True, 4).cpu().double().numpy()
    assert np.abs(lim - ref.giou3d64(c1, c2, nk, True, 4)).max() < ATOL
    assert np.abs(full - ref.giou3d64(c1, c2, nk, True)).max() < ATOL
    assert np.array_equal(lim[:, :, :4], full[:, :, :4])
    # (the rotated path also drops the intersection wherever the rectangle spanned by ground corners 1 and 3 of the
    # two boxes is empty -- the reference's `non_rot` gate -- so only some of the overlapping pairs differ)
    assert ((full - lim)[:, :, 4:] > 1e-3).sum() >= 1 and (full >= lim).all() and (lim[:, :, 4:] != 0).all()


def test_degenerate_boxes_have_their_defined_results():
    mk = lambda s, c: get_3d_box_batch_tensor(torch.tensor(s), torch.zeros(len(s)),
                                              flip_axis_to_camera_tensor(torch.tensor(c)))[None]
    boxes = mk([[1.0, 2.0, 0.5], [0.3, 0.3, 0.3], [1.0, 1.0, 0.0], [0.0, 0.0, 0.0]],
               [[10.0, 10.0, 0.5], [10.2, 10.1, 0.5], [10.0, 10.0, 0.5], [10.0, 10.0, 0.5]])
    boxes = torch.cat((boxes, torch.zeros(1, 1, 8, 3)), dim=1)            # ... and the all-zero padding box
    nk = torch.tensor([5], dtype=torch.int32)
    iou = apc.box3d_iou(boxes.cuda(), boxes.cuda()).cpu()
    assert np.abs(iou.double().numpy() - ref.box3d_iou64(boxes, boxes)).max() < ATOL
    # identical axis-aligned boxes: 1;  zero height, zero size, all zero: the denominator is not positive -> exactly 0
    assert abs(float(iou[0, 0, 0]) - 1) < ATOL and abs(float(iou[0, 1, 1]) - 1) < ATOL
    assert (iou[0, 2:, :] == 0).all() and (iou[0, :, 2:] == 0).all() and torch.isfinite(iou).all()
    for rotated in (False, True):
        g = ops.giou3d(boxes.cuda(), boxes.cuda(), nk.cuda(), rotated).cpu()
        assert torch.isfinite(g).all()
        assert np.abs(g.double().numpy() - ref.giou3d64(boxes, boxes, nk, rotated)).max() < ATOL, rotated
        # two boxes without extent enclose nothing: not `good`, exactly 0
        assert (g[0, 3:, 3:] == 0).all()
        if not rotated:
            assert abs(float(g[0, 0, 0]) - 1) < ATOL and abs(float(g[0, 1, 1]) - 1) < ATOL


def test_giou3d_and_iou_at_the_models_shapes():
    """256 queries x 64 ground-truth slots x 8 scenes, boxes of furniture size in a room that reaches 10 m"""
    g = torch.Generator().manual_seed(3)
    b, k1, k2 = 8, 256, 64
    size = lambda k: torch.rand(b, k, 3, generator=g) * 1.7 + 0.1
    ang = lambda k: (torch.rand(b, k, generator=g) * 2 - 1) * math.pi
    cen = lambda k: torch.rand(b, k, 3, generator=g) * torch.tensor([8.0, 8.0, 1.5]) + torch.tensor([2.0, 2.0, -0.7])
    c1 = get_3d_box_batch_tensor(size(k1), ang(k1), flip_axis_to_camera_tensor(cen(k1)))
    c2 = get_3d_box_batch_tensor(size(k2), ang(k2), flip_axis_to_camera_tensor(cen(k2)))
    c2[:, :16] = c1[:, :16] + 0.03
    nk = torch.tensor([64, 40, 17, 0, 64, 1, 33, 5], dtype=torch.int32)
    got = ops.giou3d(c1.cuda(), c2.cuda(), nk.cuda(), True).cpu().double().numpy()
    assert np.abs(got - ref.giou3d64(c1, c2, nk, True)).max() < ATOL
    iou = apc.box3d_iou(c1[:2].cuda(), c2[:2].cuda()).cpu().double().numpy()
    iou64 = ref.box3d_iou64(c1[:2], c2[:2])
    assert (iou64 > 0).sum() > 300 and np.abs(iou - iou64).max() < ATOL
