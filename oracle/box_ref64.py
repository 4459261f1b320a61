"""fp64 references of the box geometry and of the evaluation rules (CHECKERS for csrc/detr_kernels.cu giou3d_kernel
and the four kernels of csrc/eval_kernels.cu), written from the definitions in include/coda_detr.h and
include/coda_eval.h -- not from the kernels' arithmetic, which oracle/giou_ref.py + box_oracle.c restate in fp32.

Everything takes the fp32 inputs the kernels see and computes in fp64 (Python floats / numpy float64), so the
difference to a kernel is the kernel's rounding alone.  Box corners are (8, 3) in the order of get_3d_box: corners 0-3
one horizontal face, 4-7 the other; camera frame (x right, y down, z forward)."""
import numpy as np

EPS = 1e-8


def _np64(t):
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


# --------------------------------------------------------------------------- area of quadrilateral intersection
def _cross(ax, ay, bx, by):
    return ax * by - ay * bx


def clip_area64(rect1, rect2):
    """Area of the intersection of quadrilateral rect1 (4, 2) with CONVEX quadrilateral rect2 (4, 2).

    Sutherland-Hodgman: rect1 is cut by the four half-planes of rect2.  A point is inside a half-plane when it lies
    STRICTLY on the interior side of the edge (the rule of the reference's polygon_clip, which the kernels keep: a
    vertex exactly on a clip edge is outside).  Works for either winding of rect2; a rect2 of zero area has no
    interior.  Crossing points are found parametrically along the subject edge."""
    poly = [(float(p[0]), float(p[1])) for p in rect1]
    clip = [(float(p[0]), float(p[1])) for p in rect2]
    twice = sum(_cross(clip[i - 1][0], clip[i - 1][1], clip[i][0], clip[i][1]) for i in range(4))
    if twice == 0.0:
        return 0.0
    sign = 1.0 if twice > 0 else -1.0
    for i in range(4):
        ax, ay = clip[i - 1]
        ex, ey = clip[i][0] - ax, clip[i][1] - ay
        side = [sign * _cross(ex, ey, px - ax, py - ay) for px, py in poly]
        out = []
        for q in range(len(poly)):
            s, e = poly[q - 1], poly[q]
            ds, de = side[q - 1], side[q]
            if (de > 0) != (ds > 0):
                t = ds / (ds - de)
                out.append((s[0] + t * (e[0] - s[0]), s[1] + t * (e[1] - s[1])))
            if de > 0:
                out.append(e)
        poly = out
        if not poly:
            return 0.0
    # shoelace about the first vertex: the area does not depend on the origin, the rounding should not either
    x0, y0 = poly[0]
    acc = 0.0
    for q in range(1, len(poly) - 1):
        acc += _cross(poly[q][0] - x0, poly[q][1] - y0, poly[q + 1][0] - x0, poly[q + 1][1] - y0)
    return abs(acc) * 0.5


def _ground_rects(c):
    """(..., 8, 3) -> (..., 4, 2): corners 3, 2, 1, 0 as (x, z)."""
    return c[..., [3, 2, 1, 0], :][..., [0, 2]]


def _pair_clip_areas(r1, r2, want):
    """r1 (b, k1, 4, 2), r2 (b, k2, 4, 2), want (b, k1, k2) bool -> clip_area64 where wanted, else 0.  Pairs whose
    (x, z) bounding rectangles do not overlap have no intersection and are not clipped."""
    lo1, hi1, lo2, hi2 = r1.min(-2), r1.max(-2), r2.min(-2), r2.max(-2)
    apart = ((lo1[:, :, None] >= hi2[:, None]) | (lo2[:, None] >= hi1[:, :, None])).any(-1)
    out = np.zeros(want.shape)
    for b, i, j in zip(*np.nonzero(want & ~apart)):
        out[b, i, j] = clip_area64(r1[b, i], r2[b, j])
    return out


def _edge(c, i, j):
    return np.sqrt(((c[..., i, :] - c[..., j, :]) ** 2).sum(-1))


# --------------------------------------------------------------------------- IoU / GIoU
def box3d_iou64(c1, c2):
    """c1 (b, k1, 8, 3), c2 (b, k2, 8, 3) -> IoU (b, k1, k2) of upright boxes rotated about y (include/coda_eval.h):
    ground-plane intersection area x height overlap / (vol1 + vol2 - intersection); 0 where that denominator is
    not positive."""
    c1, c2 = _np64(c1), _np64(c2)
    area = _pair_clip_areas(_ground_rects(c1), _ground_rects(c2), np.ones((c1.shape[0], c1.shape[1], c2.shape[1]), bool))
    ymax = np.minimum(c1[:, :, None, 0, 1], c2[:, None, :, 0, 1])
    ymin = np.maximum(c1[:, :, None, 4, 1], c2[:, None, :, 4, 1])
    inter = area * np.maximum(ymax - ymin, 0.0)
    v1 = _edge(c1, 0, 1) * _edge(c1, 1, 2) * _edge(c1, 0, 4)
    v2 = _edge(c2, 0, 1) * _edge(c2, 1, 2) * _edge(c2, 0, 4)
    den = v1[:, :, None] + v2[:, None, :] - inter
    return np.where(den > 0, inter / np.where(den > 0, den, 1.0), 0.0)


def giou3d64(c1, c2, nums_k2, rotated, rot_k2_limit=None):
    """Generalised IoU (b, k1, k2) as include/coda_detr.h defines it (generalized_box3d_iou_tensor of the reference):

      height     = overlap of the two y ranges, >= 0
      non_rot    = overlap of the (x, z) rectangles spanned by ground corners 1 and 3 -- the true intersection area of
                   axis-aligned boxes
      inter area = non_rot if not rotated; else the polygon intersection where non_rot != 0 and column < rot_k2_limit,
                   0 elsewhere
      vol        = max(product of the three edge lengths, each sqrt(max(|e|^2, 1e-6)), EPS)
      union      = max(vol1 + vol2 - inter area * height, EPS),  enclosing = axis-aligned hull of the 16 corners
      giou       = inter / union - (1 - union / enclosing)   where enclosing > 2 EPS and vol1 + vol2 > 4 EPS, else 0
      columns >= nums_k2[b] are 0."""
    c1, c2 = _np64(c1), _np64(c2)
    b, k1, k2 = c1.shape[0], c1.shape[1], c2.shape[1]
    lim = k2 if rot_k2_limit is None else int(rot_k2_limit)
    nk = np.asarray(nums_k2.detach().cpu().numpy() if hasattr(nums_k2, "detach") else nums_k2).astype(np.int64)
    ymax = np.minimum(c1[:, :, None, 0, 1], c2[:, None, :, 0, 1])
    ymin = np.maximum(c1[:, :, None, 4, 1], c2[:, None, :, 4, 1])
    height = np.maximum(ymax - ymin, 0.0)
    r1, r2 = _ground_rects(c1), _ground_rects(c2)
    lt = np.maximum(r1[:, :, None, 1], r2[:, None, :, 1])
    rb = np.minimum(r1[:, :, None, 3], r2[:, None, :, 3])
    wh = np.maximum(rb - lt, 0.0)
    non_rot = wh[..., 0] * wh[..., 1]
    live = np.arange(k2)[None, None, :] < nk[:, None, None]
    if rotated:
        want = (non_rot != 0) & live & (np.arange(k2)[None, None, :] < lim)
        area = _pair_clip_areas(r1, r2, want)
    else:
        area = non_rot
    lo = np.minimum(c1.min(-2)[:, :, None], c2.min(-2)[:, None])
    hi = np.maximum(c1.max(-2)[:, :, None], c2.max(-2)[:, None])
    enclosing = np.prod(hi - lo, axis=-1)

    def vol(c):
        def e(i, j):
            return np.sqrt(np.maximum(((c[..., i, :] - c[..., j, :]) ** 2).sum(-1), 1e-6))
        return np.maximum(e(0, 1) * e(1, 2) * e(0, 4), EPS)

    sum_vols = vol(c1)[:, :, None] + vol(c2)[:, None, :]
    good = (enclosing > 2 * EPS) & (sum_vols > 4 * EPS)
    inter = area * height
    union = np.maximum(sum_vols - inter, EPS)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = inter / union - (1.0 - union / enclosing)
    return np.where(good & live, g, 0.0)


# --------------------------------------------------------------------------- NMS
def nms3d_ref(corners, score, cls, valid, thresh, old_type=False):
    """Sequential greedy NMS of include/coda_eval.h for ONE scene: corners (k, 8, 3), score (k), cls (k) or None,
    valid (k) -> (keep (k) bool, margin).

    Candidates are the valid boxes whose score is not NaN, visited in descending score order, among equal scores the
    higher index first.  A visited box that is still alive is kept and drops every later candidate j with
    inter / (vol_i + vol_j - inter) > thresh (old_type: inter / vol_j) on the axis-aligned extents -- of its own
    class only when cls is given.  0 / 0 compares false: a box of zero volume is never dropped.
    margin = the smallest |overlap - thresh| over all decisions taken on a non-zero intersection: where it is below
    the rounding of an fp32 overlap, an fp32 implementation may rightly decide otherwise."""
    c = _np64(corners)
    s = _np64(score)
    k = c.shape[0]
    ok = np.asarray(valid.cpu().numpy() if hasattr(valid, "cpu") else valid).astype(bool) & ~np.isnan(s)
    kl = None if cls is None else np.asarray(cls.cpu().numpy() if hasattr(cls, "cpu") else cls)
    lo, hi = c.min(1), c.max(1)
    vol = np.prod(hi - lo, axis=1)
    cand = [i for i in range(k) if ok[i]]
    cand.sort(key=lambda i: (-s[i], -i))
    order = np.array(cand, dtype=np.int64)
    alive = np.ones(len(order), bool)
    keep = np.zeros(k, bool)
    margin = np.inf
    for a, i in enumerate(order):
        if not alive[a]:
            continue
        keep[i] = True
        rest = order[a + 1:]
        if rest.size == 0:
            break
        ext = np.maximum(np.minimum(hi[i], hi[rest]) - np.maximum(lo[i], lo[rest]), 0.0)
        inter = ext.prod(1)
        with np.errstate(divide="ignore", invalid="ignore"):
            o = inter / vol[rest] if old_type else inter / (vol[i] + vol[rest] - inter)
        if kl is not None:
            o = np.where(kl[rest] == kl[i], o, 0.0)
            inter = np.where(kl[rest] == kl[i], inter, 0.0)
        judged = alive[a + 1:] & (inter > 0) & ~np.isnan(o)
        if judged.any():
            margin = min(margin, float(np.abs(o[judged] - thresh).min()))
        with np.errstate(invalid="ignore"):
            alive[a + 1:] &= ~(o > thresh)
    return keep, margin


# --------------------------------------------------------------------------- points inside boxes
def points_in_boxes_coords(corners_camera, points_depth):
    """corners (k, 8, 3) camera frame, points (n, >=3) depth frame -> (k, n, 3) coordinates of every point in every
    box's edge frame (origin corner 0, axes the edges 0-1, 0-3, 0-4), as fractions of the edge: inside = [0, 1]^3.
    NaN along an edge of length zero."""
    c = _np64(corners_camera)
    p = _np64(points_depth)[:, :3]
    d = np.stack((c[..., 0], c[..., 2], -c[..., 1]), axis=-1)       # camera (x, y, z) -> depth (x, z, -y)
    o = d[:, 0]
    axes = np.stack((d[:, 1] - o, d[:, 3] - o, d[:, 4] - o), axis=1)   # (k, 3 edges, 3)
    rel = p[None, :, :] - o[:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.einsum("kne,kae->kna", rel, axes) / (axes ** 2).sum(-1)[:, None, :]


def points_in_boxes_ref(corners_camera, points_depth):
    """(k, 8, 3), (n, >=3) -> (k) number of points inside each box, faces inclusive; a box with an edge of length
    zero holds no point (include/coda_eval.h)."""
    t = points_in_boxes_coords(corners_camera, points_depth)
    with np.errstate(invalid="ignore"):
        return ((t >= 0) & (t <= 1)).all(-1).sum(-1).astype(np.int64)


# --------------------------------------------------------------------------- VOC matching
def eval_match_ref(iou, scores, det_mask, gt_cls, gt_present, thresh):
    """The sequential rule of include/coda_eval.h (reference utils/eval_det.py:110-146): iou (b, k, g), scores
    (b, k, c), det_mask (b, k), gt_cls (b, g), gt_present (b, g) -> tp (b, c, k) bool.  Per scene and class, the
    detections in play (det_mask, score neither -inf nor NaN) are visited in descending score order, equal scores
    by ascending index; each looks up the present ground-truth box of the class with the largest IoU (the first one
    among equals) and is a true positive if that IoU > thresh and the box is not claimed yet -- it then claims it."""
    io, sc = np.asarray(iou), np.asarray(scores)
    dm, gc, pr = np.asarray(det_mask).astype(bool), np.asarray(gt_cls), np.asarray(gt_present).astype(bool)
    b, k, c = sc.shape
    exp = np.zeros((b, c, k), bool)
    for i in range(b):
        for cc in range(c):
            gts = [q for q in range(pr.shape[1]) if pr[i, q] and gc[i, q] == cc]
            if not gts:
                continue
            claimed = set()
            for j in np.argsort(-sc[i, :, cc], kind="stable"):
                if not dm[i, j] or not sc[i, j, cc] > -np.inf:
                    continue
                m = gts[int(np.argmax([io[i, j, q] for q in gts]))]
                if io[i, j, m] > thresh and m not in claimed:
                    claimed.add(m)
                    exp[i, cc, j] = True
    return exp
