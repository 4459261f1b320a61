"""Stage-2 candidate selection (coda_novel_candidates, csrc/discovery_kernels.cu) against the step-by-step restatement
of the reference loop (oracle/discovery_ref.py: torchvision.ops.nms, cal_iou, the objectness threshold), exactly, at
the edges of its shapes (q on both sides of a 32-bit word, of the 256-thread block and of MAXQ; cap from 1 to past
q; no ground truth), on its three decision boundaries hit exactly (2-D IoU == nms_iou, 3-D IoU == gt_iou,
objectness == save_objectness), on ties, and on non-finite scores: NaN ranks above every number like in
torchvision's stable descending sort.  Every call writes between guard words, and every result is checked to be a
list of distinct box indices padded with -1.  tests/test_crop_discovery_paths_cpu.py checks that the shape cases
reach every edge."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import discovery_ref
from coda_neurips2023_b200 import ops
from coda_neurips2023_b200._lib import lib

pytestmark = pytest.mark.gpu

QS = (1, 31, 32, 33, 128, 255, 256, 257, 1000, 1024)
GS = (0, 1, 64)
CAPS = ("1", "32", "q", "q+5")
MODEL_SHAPE = (8, 128, 64, 32)         # scenes, queries, ground-truth slots, capacity of the stage-2 step
REFUSED = ((1, 1025, 4, 8), (1, 16, 4, 0))
THRESHOLDS = (0.25, 0.25, 0.4)         # nms_iou, gt_iou, save_objectness of the step
GUARD = 16
SENTINEL = -12345


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    pass


def cap_of(spec: str, q: int) -> int:
    return {"1": 1, "32": 32, "q": q, "q+5": q + 5}[spec]


def _corners(lo, hi):
    """(..., 3) lower / upper corners -> (..., 8, 3) corners of the axis-aligned box"""
    sel = torch.tensor(list(itertools.product((0, 1), repeat=3)), dtype=torch.bool)
    return torch.where(sel, hi.unsqueeze(-2), lo.unsqueeze(-2))


def random_case(b, q, g, seed):
    """boxes in a 600 x 600 image with exact duplicates and a score tie, 3-D boxes overlapping the ground truth
    about as often as in a scene"""
    gen = torch.Generator().manual_seed(seed)
    xy = torch.randint(0, 600, (b, q, 2), generator=gen)
    wh = torch.randint(1, 250, (b, q, 2), generator=gen)
    boxes = torch.cat((xy, xy + wh), dim=-1).to(torch.int32)
    if q >= 16:
        boxes[:, : q // 8] = boxes[:, q // 8: 2 * (q // 8)]
    valid = torch.rand(b, q, generator=gen) > 0.15
    obj = torch.rand(b, q, generator=gen)
    if q >= 7:
        obj[:, 5] = obj[:, 6]
    ctr = torch.rand(b, q, 3, generator=gen) * 4
    half = torch.rand(b, q, 3, generator=gen) * 0.8 + 0.1
    gctr = torch.rand(b, max(g, 1), 3, generator=gen) * 4
    ghalf = torch.rand(b, max(g, 1), 3, generator=gen) * 0.8 + 0.1
    gt = _corners(gctr - ghalf, gctr + ghalf)[:, :g]
    present = (torch.rand(b, max(g, 1), generator=gen) > 0.3).float()[:, :g]
    return boxes, valid, obj, _corners(ctr - half, ctr + half), gt, present


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def run_kernel(boxes, valid, obj, pred, gt, present, cap, thr=THRESHOLDS):
    """the C entry point, with cand_idx and cand_count between guard words -> (status, cand (b, cap), count (b, 2))"""
    b, q, _ = boxes.shape
    g = gt.shape[1]
    dev = "cuda"
    bx, vd = boxes.to(torch.int32).contiguous().to(dev), valid.to(torch.uint8).contiguous().to(dev)
    ob, pc = obj.float().contiguous().to(dev), pred.float().contiguous().to(dev)
    gc, gp = gt.float().contiguous().to(dev), present.float().contiguous().to(dev)
    cbuf = torch.full((b * max(cap, 0) + 2 * GUARD,), SENTINEL, dtype=torch.int32, device=dev)
    nbuf = torch.full((2 * b + 2 * GUARD,), SENTINEL, dtype=torch.int32, device=dev)
    i, f = ctypes.c_int, ctypes.c_float
    st = lib().coda_novel_candidates(i(b), i(q), i(g), i(cap), _p(bx), _p(vd), _p(ob), _p(pc), _p(gc), _p(gp),
                                     f(thr[0]), f(thr[1]), f(thr[2]), ctypes.c_void_p(cbuf[GUARD:].data_ptr()),
                                     ctypes.c_void_p(nbuf[GUARD:].data_ptr()),
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    for buf, n in ((cbuf, b * max(cap, 0)), (nbuf, 2 * b)):
        assert (buf[:GUARD] == SENTINEL).all() and (buf[GUARD + n:] == SENTINEL).all(), "a guard word changed"
    if st != 0:
        assert (cbuf == SENTINEL).all() and (nbuf == SENTINEL).all(), "a refused call wrote"
    return st, cbuf[GUARD:GUARD + b * max(cap, 0)].view(b, max(cap, 0)).cpu(), nbuf[GUARD:GUARD + 2 * b].view(b, 2).cpu()


def check_case(boxes, valid, obj, pred, gt, present, caps, thr=THRESHOLDS):
    """kernel == oracle for every capacity in `caps`, and the result is a -1 padded list of distinct indices"""
    q = boxes.shape[1]
    full_idx, full_cnt = discovery_ref.novel_candidates_ref(boxes, valid, obj, pred, gt, present, *thr, q)
    for cap in caps:
        st, cand, cnt = run_kernel(boxes, valid, obj, pred, gt, present, cap, thr)
        assert st == 0
        exp_cnt = torch.stack((full_cnt[:, 1].clamp(max=cap), full_cnt[:, 1]), 1)
        exp_idx = torch.full((boxes.shape[0], cap), -1, dtype=torch.int32)
        exp_idx[:, : min(cap, q)] = full_idx[:, : min(cap, q)]
        assert torch.equal(cnt, exp_cnt), (cap, cnt, exp_cnt)
        assert torch.equal(cand, exp_idx), cap
        assert ((cand >= -1) & (cand < q)).all()
        assert torch.equal(cnt[:, 0], cnt[:, 1].clamp(max=cap))
        for row, n in zip(cand, cnt[:, 0].tolist()):
            kept = row[:n]
            assert (kept >= 0).all() and len(set(kept.tolist())) == n and (row[n:] == -1).all()
    return full_idx, full_cnt


@pytest.mark.parametrize("q", QS)
@pytest.mark.parametrize("g", GS)
def test_shapes_match_reference(q, g):
    """every q edge, with and without ground truth, at capacities 1, 32, q and q + 5"""
    case = random_case(2, q, g, seed=q * 7 + g)
    check_case(*case, [cap_of(c, q) for c in CAPS])


def test_model_shape_through_ops():
    b, q, g, cap = MODEL_SHAPE
    boxes, valid, obj, pred, gt, present = random_case(b, q, g, seed=99)
    exp_idx, exp_cnt = discovery_ref.novel_candidates_ref(boxes, valid, obj, pred, gt, present, *THRESHOLDS, cap)
    cand, cnt = ops.novel_candidates(boxes.cuda(), valid.cuda(), obj.cuda(), pred.cuda(), gt.cuda(), present.cuda(),
                                     *THRESHOLDS, cap)
    assert torch.equal(cnt.cpu(), exp_cnt) and torch.equal(cand.cpu(), exp_idx)
    check_case(boxes, valid, obj, pred, gt, present, [cap])


@pytest.mark.parametrize("b,q,g,cap", REFUSED)
def test_refused_arguments(b, q, g, cap):
    boxes, valid, obj, pred, gt, present = random_case(b, q, g, seed=5)
    st, _, _ = run_kernel(boxes, valid, obj, pred, gt, present, cap)
    assert st == -1                                      # CODA_EINVAL
    with pytest.raises(RuntimeError):
        ops.novel_candidates(boxes.cuda(), valid.cuda(), obj.cuda(), pred.cuda(), gt.cuda(), present.cuda(),
                             *THRESHOLDS, cap)


def _far_3d(q):
    """3-D boxes of every query far from the ground truth of _one_gt"""
    lo = torch.full((1, q, 3), 50.0) + torch.arange(q, dtype=torch.float32).view(1, q, 1) * 3
    return _corners(lo, lo + 1)


def _one_gt():
    return _corners(torch.zeros(1, 1, 3), torch.ones(1, 1, 3)), torch.ones(1, 1)


def test_2d_iou_exactly_at_threshold_is_kept():
    """[0,0,10,10] and [6,0,16,10] overlap with IoU 0.25 exactly: both survive; [5,0,15,10] (IoU 1/3) is suppressed"""
    boxes = torch.tensor([[[0, 0, 10, 10], [6, 0, 16, 10], [5, 0, 15, 10]]], dtype=torch.int32)
    obj = torch.tensor([[0.9, 0.8, 0.7]])
    gt, present = _one_gt()
    idx, cnt = check_case(boxes, torch.ones(1, 3, dtype=torch.bool), obj, _far_3d(3), gt, present, [3])
    assert idx[0, :2].tolist() == [0, 1] and cnt[0].tolist() == [2, 2]


def test_3d_iou_exactly_at_threshold_is_kept():
    """the ground truth [0,1]^3 inside the prediction [0,2]x[0,2]x[0,1]: IoU 1/4 exactly, kept; inside
    [0,2]x[0,1.75]x[0,1] (IoU 2/7) rejected"""
    boxes = torch.tensor([[[0, 0, 10, 10], [100, 100, 110, 110], [200, 200, 210, 210]]], dtype=torch.int32)
    lo = torch.zeros(1, 3, 3)
    hi = torch.tensor([[[2.0, 2.0, 1.0], [2.0, 1.75, 1.0], [60.0, 60.0, 60.0]]])
    lo[0, 2] = 50.0
    gt, present = _one_gt()
    idx, cnt = check_case(boxes, torch.ones(1, 3, dtype=torch.bool), torch.tensor([[0.9, 0.8, 0.7]]),
                          _corners(lo, hi), gt, present, [3])
    assert idx[0, :2].tolist() == [0, 2] and cnt[0].tolist() == [2, 2]


def test_objectness_exactly_at_threshold_is_kept():
    below = float(np.nextafter(np.float32(0.75), np.float32(0)))
    boxes = torch.tensor([[[0, 0, 10, 10], [100, 100, 110, 110], [200, 200, 210, 210]]], dtype=torch.int32)
    obj = torch.tensor([[0.75, below, 0.9]])
    gt, present = _one_gt()
    idx, cnt = check_case(boxes, torch.ones(1, 3, dtype=torch.bool), obj, _far_3d(3), gt, present, [3],
                          (0.25, 0.25, 0.75))
    assert idx[0, :2].tolist() == [2, 0] and cnt[0].tolist() == [2, 2]


def _tie_cases():
    q, g = 40, 8
    out = {}
    boxes, valid, obj, pred, gt, present = random_case(3, q, g, seed=21)
    out["all scores equal"] = (boxes, valid, torch.full_like(obj, 0.5), pred, gt, present)
    signed = torch.where(torch.arange(q) % 2 == 0, torch.tensor(-0.0), torch.tensor(0.0)).expand(3, q).clone()
    out["-0.0 and +0.0"] = (boxes, torch.ones_like(valid), signed, pred, gt, present, (0.25, 0.25, 0.0))
    dup = boxes.clone()
    dup[:, 1::2] = dup[:, 0::2]
    out["duplicate boxes"] = (dup, valid, obj, pred, gt, present)
    out["every box given up"] = (boxes, torch.zeros_like(valid), obj, pred, gt, present)
    out["no ground truth present"] = (boxes, valid, obj, pred, gt, torch.zeros_like(present))
    return out


@pytest.mark.parametrize("name", list(_tie_cases()))
def test_ties_and_empty_sets(name):
    case = _tie_cases()[name]
    thr = case[6] if len(case) > 6 else THRESHOLDS
    idx, cnt = check_case(*case[:6], [1, 40, 45], thr)
    if name == "every box given up":
        assert (cnt == 0).all() and (idx == -1).all()


def _nonfinite_cases():
    q, g = 64, 8
    nan, inf = float("nan"), float("inf")
    out = {}
    for name, where, value in (("NaN first", [0], nan), ("NaN last", [q - 1], nan),
                               ("NaN on several", [3, 9, 10, 40, 63], nan), ("NaN everywhere", list(range(q)), nan),
                               ("+inf on several", [2, 7, 50], inf), ("-inf and NaN", [4, 5], None)):
        boxes, valid, obj, pred, gt, present = random_case(2, q, g, seed=len(out) + 40)
        obj = obj.clone()
        if value is None:
            obj[:, 4], obj[:, 5] = -inf, nan
        else:
            obj[:, where] = value
        out[name] = (boxes, valid, obj, pred, gt, present)
    return out


@pytest.mark.parametrize("name", list(_nonfinite_cases()))
def test_nonfinite_scores_rank_like_torchvision(name):
    """NaN ranks above every number, ties by index: the emitted list is the oracle's, a prefix of a permutation"""
    check_case(*_nonfinite_cases()[name], [1, 16, 64, 69])
