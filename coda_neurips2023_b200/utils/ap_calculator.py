"""Average-precision evaluation of the detector on the device (mirror of reference utils/ap_calculator.py:
`get_ap_config_dict`, `parse_predictions`, `APCalculator` with the same constructor, `step_meter` / `step` /
`compute_metrics` / `metrics_to_str` / `metrics_to_dict` / `reset`, the same result-dict keys).

The reference walks every predicted box on the host: a scipy Delaunay hull test per box for `remove_empty_box`
(ap_calculator.py:808-835), numpy NMS per scene (:868-941, utils/nms.py), Python tuples per (class, box), then
utils/eval_det.py computes the IoU of every (detection, ground truth) pair one polygon clip at a time.  Here a step is
five kernel launches (include/coda_eval.h) on the batch as it leaves the model -- nothing is copied to the host until
`compute_metrics`, which only sees (score, true-positive flag) pairs:

    points_in_boxes -> non-empty mask | nms3d (same-class / class-agnostic) | box3d_iou (B, K, G) |
    eval_match per IoU threshold -> tp (B, C, K)

`compute_metrics` compacts what the steps accumulated into one record per (scene, box, class) detection
(`coda_eval_records`), sorts the records by (class, score descending, scene and box), and computes precision / recall /
VOC AP of every class and IoU threshold in one launch (`coda_eval_ap`) as utils/eval_det.py:147-162 + voc_ap (:23-55)
do.  Records are what data-parallel ranks exchange: a rank-local calculator scores only its own scenes and merges the
other ranks' records in `compute_metrics`, instead of gathering every point cloud and output before each step.
"""
from __future__ import annotations

import ctypes
from collections import OrderedDict
from typing import NamedTuple

import numpy as np
import torch

from .._lib import check, lib, ptr, stream_of


def _i(v):
    return ctypes.c_int(int(v))


def _f(v):
    return ctypes.c_float(float(v))


# --------------------------------------------------------------------------- kernel wrappers
def points_in_boxes(corners_camera: torch.Tensor, points_depth: torch.Tensor) -> torch.Tensor:
    """(B, K, 8, 3) camera-frame corners, (B, N, >=3) depth-frame points -> (B, K) int32 points inside each box."""
    if not corners_camera.is_cuda:
        raise RuntimeError("points_in_boxes: CPU not supported")
    c = corners_camera.detach().float().contiguous()
    p = points_depth.detach().float().contiguous()
    b, k = c.shape[:2]
    out = torch.empty((b, k), dtype=torch.int32, device=c.device)
    with torch.cuda.device(c.device):
        st = lib().coda_points_in_boxes(_i(b), _i(k), _i(p.shape[1]), _i(p.shape[2]), ptr(c), ptr(p), ptr(out),
                                        stream_of(c))
    check(st, "points_in_boxes")
    return out


def nms3d(corners: torch.Tensor, score: torch.Tensor, valid: torch.Tensor, iou_thresh: float, cls=None,
          old_type: bool = False) -> torch.Tensor:
    """Greedy 3-D NMS per scene on axis-aligned extents: (B, K, 8, 3), (B, K), (B, K) bool -> keep (B, K) bool.
    cls (B, K) int: only boxes of the same class suppress each other (utils/nms.py:120-162)."""
    if not corners.is_cuda:
        raise RuntimeError("nms3d: CPU not supported")
    c = corners.detach().float().contiguous()
    s = score.detach().float().contiguous()
    v = valid.to(torch.uint8).contiguous()
    kl = None if cls is None else cls.to(torch.int32).contiguous()
    b, k = c.shape[:2]
    keep = torch.empty((b, k), dtype=torch.uint8, device=c.device)
    with torch.cuda.device(c.device):
        st = lib().coda_nms3d(_i(b), _i(k), ptr(c), ptr(s), ptr(kl), ptr(v), _f(iou_thresh), _i(1 if old_type else 0),
                              ptr(keep), stream_of(c))
    check(st, "nms3d")
    return keep.bool()


def box3d_iou(corners1: torch.Tensor, corners2: torch.Tensor) -> torch.Tensor:
    """(B, K1, 8, 3), (B, K2, 8, 3) -> IoU (B, K1, K2) of upright rotated boxes (utils/box_util.py:156-183)."""
    if not corners1.is_cuda:
        raise RuntimeError("box3d_iou: CPU not supported")
    c1 = corners1.detach().float().contiguous()
    c2 = corners2.detach().float().contiguous()
    b, k1, k2 = c1.shape[0], c1.shape[1], c2.shape[1]
    out = torch.zeros((b, k1, k2), dtype=torch.float32, device=c1.device)
    with torch.cuda.device(c1.device):
        st = lib().coda_box3d_iou(_i(b), _i(k1), _i(k2), ptr(c1), ptr(c2), ptr(out), stream_of(c1))
    check(st, "box3d_iou")
    return out


def eval_match(iou: torch.Tensor, scores: torch.Tensor, det_mask: torch.Tensor, gt_cls: torch.Tensor,
               gt_present: torch.Tensor, iou_thresh: float) -> torch.Tensor:
    """iou (B, K, G), scores (B, K, C) (-inf = no detection of that class), det_mask (B, K), gt_cls (B, G),
    gt_present (B, G) -> tp (B, C, K) bool (utils/eval_det.py:110-146 per scene and class)."""
    if not scores.is_cuda:
        raise RuntimeError("eval_match: CPU not supported")
    b, k, c = scores.shape
    g = gt_cls.shape[1]
    tp = torch.zeros((b, c, k), dtype=torch.uint8, device=scores.device)
    # converted copies must outlive the launch: a temporary freed between two pointer extractions hands its block to
    # the next temporary
    io, sc = iou.float().contiguous(), scores.float().contiguous()
    dm, gc, gp = (det_mask.to(torch.uint8).contiguous(), gt_cls.to(torch.int32).contiguous(),
                  gt_present.to(torch.uint8).contiguous())
    with torch.cuda.device(scores.device):
        st = lib().coda_eval_match(_i(b), _i(k), _i(g), _i(c), ptr(io), ptr(sc), ptr(dm), ptr(gc), ptr(gp),
                                   _f(iou_thresh), ptr(tp), stream_of(scores))
    check(st, "eval_match")
    return tp.bool()


class EvalRecords(NamedTuple):
    """One record per (scene, box, class) detection: class int32, score fp32, global position int64 (scene x K + box,
    the order that breaks score ties), tp int32 (bit t = true positive at IoU threshold t)."""
    cls: torch.Tensor
    score: torch.Tensor
    pos: torch.Tensor
    tp: torch.Tensor

    def __len__(self):
        return self.cls.shape[0]


def eval_records(scores: list, det_masks: list, tps: list, scene_bases: list) -> EvalRecords:
    """Compacts accumulated steps -- scores (B, K, C) f32 (-inf / NaN = no detection), det_mask (B, K) bool,
    tp (T, B, C, K) bool and the global number of each step's first scene -- into detection records, in no
    particular order."""
    dev = scores[0].device
    cap = sum(s.numel() for s in scores)
    rec = EvalRecords(torch.empty(cap, dtype=torch.int32, device=dev), torch.empty(cap, dtype=torch.float32, device=dev),
                      torch.empty(cap, dtype=torch.int64, device=dev), torch.empty(cap, dtype=torch.int32, device=dev))
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        for s, m, t, base in zip(scores, det_masks, tps, scene_bases):
            b, k, c = s.shape
            s, m, t = s.float().contiguous(), _bytes(m), _bytes(t)
            st = lib().coda_eval_records(_i(b), _i(k), _i(c), _i(t.shape[0]), ctypes.c_longlong(int(base)), ptr(s),
                                         ptr(m), ptr(t), ptr(counter), _i(cap), ptr(rec.cls), ptr(rec.score),
                                         ptr(rec.pos), ptr(rec.tp), stream_of(s))
            check(st, "eval_records")
    n = int(counter.item())
    if n > cap:
        raise RuntimeError(f"eval_records: {n} records for a capacity of {cap}")
    return EvalRecords(*(f[:n] for f in rec))


def _bytes(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t.view(torch.uint8) if t.dtype == torch.bool else t.to(torch.uint8)


def pack_records(rec: EvalRecords) -> torch.Tensor:
    """Records as one (n, 5) int32 block for an exchange between ranks: class, score bits, position (low word, high
    word), tp mask."""
    pos = rec.pos.long()
    return torch.stack([rec.cls.int(), rec.score.float().view(torch.int32), (pos & 0xFFFFFFFF).int(),
                        (pos >> 32).int(), rec.tp.int()], dim=1)


def unpack_records(block: torch.Tensor) -> EvalRecords:
    """Inverse of `pack_records`, for a block of any strides (a row slice of a padded exchange buffer)."""
    block = block.to(torch.int32)
    pos = (block[:, 3].long() << 32) | (block[:, 2].long() & 0xFFFFFFFF)
    return EvalRecords(block[:, 0].contiguous(), block[:, 1].contiguous().view(torch.float32), pos.contiguous(),
                       block[:, 4].contiguous())


def merge_records(parts: list) -> EvalRecords:
    """The records of several ranks as one set (the order is fixed later by `sort_records`)."""
    return EvalRecords(*(torch.cat(f) for f in zip(*parts)))


def sort_records(rec: EvalRecords) -> EvalRecords:
    """Sorted by (class ascending, score descending, global position ascending): what a stable descending argsort
    of each class's scores over the step-ordered (scene, box) rows gives."""
    order = torch.sort(rec.pos, stable=True).indices
    rec = EvalRecords(*(f[order] for f in rec))
    # fp32 bits -> an unsigned key that ascends with the score, then flipped so that it descends
    score = torch.where(rec.score == 0, torch.zeros_like(rec.score), rec.score)      # -0 ties with +0
    u = score.view(torch.int32).long() & 0xFFFFFFFF
    asc = torch.where(u >= 0x80000000, u ^ 0xFFFFFFFF, u | 0x80000000)
    key = (rec.cls.long() << 32) | (0xFFFFFFFF - asc)
    order = torch.sort(key, stable=True).indices
    return EvalRecords(*(f[order] for f in rec))


def eval_ap(rec: EvalRecords, ncls: int, nthr: int, npos: torch.Tensor, curves: bool = False):
    """Per (threshold, class) VOC AP, last precision and last recall, (T, C) fp64 each, from records sorted by
    `sort_records` and the per-class ground-truth counts npos (C,); with curves=True also the (T, 4, N) cumulative TP,
    cumulative FP, recall and precision of every record.  Returns (ap, last_prec, last_rec, per-class record counts
    (C,) int64, curves or None)."""
    dev = npos.device
    counts = torch.bincount(rec.cls.long(), minlength=ncls) if len(rec) else torch.zeros(ncls, dtype=torch.int64,
                                                                                       device=dev)
    offsets = torch.zeros(ncls + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=offsets[1:])
    npos = npos.to(torch.int64).contiguous()
    tp = rec.tp.contiguous()
    ap, last_prec, last_rec = (torch.empty((nthr, ncls), dtype=torch.float64, device=dev) for _ in range(3))
    cur = torch.empty((nthr, 4, len(rec)), dtype=torch.float64, device=dev) if curves else None
    with torch.cuda.device(dev):
        st = lib().coda_eval_ap(_i(ncls), _i(nthr), ctypes.c_longlong(len(rec)), ptr(offsets), ptr(tp), ptr(npos),
                                ptr(ap), ptr(last_prec), ptr(last_rec), ptr(cur), stream_of(npos))
    check(st, "eval_ap")
    return ap, last_prec, last_rec, counts, cur


class RankState(NamedTuple):
    """What a calculator has accumulated, in the form ranks exchange: detection records, ground-truth boxes per class
    (C,) int64, first occurrence of each class among the predictions / the ground truth (C,) int64 (int64 max = never),
    and the batch size of every step."""
    records: EvalRecords
    gt_count: torch.Tensor
    first_pred: torch.Tensor
    first_gt: torch.Tensor
    batch_sizes: list


def _check_batch_sizes(per_rank: list) -> None:
    if any(list(s) != list(per_rank[0]) for s in per_rank[1:]):
        raise ValueError("data-parallel evaluation needs every rank to hold the same number of scenes at every step; "
                         f"per-rank batch sizes: {[list(s) for s in per_rank]}")


def merge_rank_states(states: list) -> RankState:
    """The states of W rank-local calculators (rank order) as the state of one calculator that saw every rank's
    scenes: records merged, ground-truth counts summed, first occurrences reduced by minimum.  Raises ValueError when
    the ranks' batch sizes differ at some step (the scene numbering assumes they do not)."""
    _check_batch_sizes([s.batch_sizes for s in states])
    live = [s for s in states if s.gt_count is not None]
    if not live:
        return states[0]
    return RankState(merge_records([s.records for s in live]), torch.stack([s.gt_count for s in live]).sum(0),
                     torch.stack([s.first_pred for s in live]).amin(0), torch.stack([s.first_gt for s in live]).amin(0),
                     list(states[0].batch_sizes))


# --------------------------------------------------------------------------- prediction parsing
def get_ap_config_dict(remove_empty_box=True, use_3d_nms=True, nms_iou=0.25, use_old_type_nms=False, cls_nms=True,
                       per_class_proposal=True, use_cls_confidence_only=False, conf_thresh=0.05, no_nms=False,
                       dataset_config=None):
    """Default mAP evaluation settings (reference utils/ap_calculator.py:1021-1051)."""
    return {
        "remove_empty_box": remove_empty_box, "use_3d_nms": use_3d_nms, "nms_iou": nms_iou,
        "use_old_type_nms": use_old_type_nms, "cls_nms": cls_nms, "per_class_proposal": per_class_proposal,
        "use_cls_confidence_only": use_cls_confidence_only, "conf_thresh": conf_thresh, "no_nms": no_nms,
        "dataset_config": dataset_config,
    }


@torch.no_grad()
def select_detections(predicted_boxes, sem_cls_probs, objectness_probs, point_cloud, config_dict):
    """Device form of parse_predictions (reference :777-1018): returns
        det_mask (B, K) bool   -- boxes that survive the empty-box filter, NMS and the objectness threshold,
        scores   (B, K, C) f32 -- the confidence of box j AS a detection of class c; -inf where box j is no
                                   detection of class c (only the per-class-proposal mode scores every class).
    """
    corners = predicted_boxes.detach().float()
    probs = sem_cls_probs.detach().float()
    obj = objectness_probs.detach().float()
    b, k = obj.shape
    ncls = probs.shape[-1]
    pred_cls = probs.argmax(-1)
    nonempty = torch.ones((b, k), dtype=torch.bool, device=obj.device)
    if config_dict["remove_empty_box"]:
        cnt = points_in_boxes(corners, point_cloud[..., :3])
        # an all-zero box is dropped outright (:822-823), the others need five points inside
        nonzero = (corners.amax(dim=(2, 3)) >= 1e-32) | (corners.amin(dim=(2, 3)) <= -1e-32)
        nonempty = nonzero & (cnt >= 5)
        # a scene whose boxes are all empty keeps its most object-like box (:837-838)
        none = ~nonempty.any(dim=1, keepdim=True)
        best = torch.nn.functional.one_hot(obj.argmax(dim=1), k).bool()
        nonempty = nonempty | (none & best)
    if config_dict.get("no_nms"):
        pred_mask = nonempty
    elif not config_dict["use_3d_nms"]:
        # bird's-eye-view NMS (:845-874): the same greedy rule on the (x, z) extents -- flatten the height
        flat = corners.clone()
        flat[..., 1] = flat[..., 1] * 0 + (torch.arange(8, device=flat.device) >= 4).float().view(1, 1, 8)
        pred_mask = nms3d(flat, obj, nonempty, config_dict["nms_iou"], None, config_dict["use_old_type_nms"])
    else:
        pred_mask = nms3d(corners, obj, nonempty, config_dict["nms_iou"],
                          pred_cls if config_dict["cls_nms"] else None, config_dict["use_old_type_nms"])
    det_mask = pred_mask & (obj > config_dict["conf_thresh"])
    if config_dict["per_class_proposal"]:
        assert config_dict["use_cls_confidence_only"] is False
        scores = probs * obj.unsqueeze(-1)
    else:
        own = torch.nn.functional.one_hot(pred_cls, ncls).bool()
        val = probs.gather(-1, pred_cls.unsqueeze(-1)) if config_dict["use_cls_confidence_only"] else obj.unsqueeze(-1)
        scores = torch.where(own, val.expand(-1, -1, ncls), torch.full_like(probs, float("-inf")))
    return det_mask, scores


def parse_predictions(predicted_boxes, sem_cls_probs, objectness_probs, point_cloud, config_dict):
    """The reference's return format -- per scene a list of (class, corners (8, 3) numpy, score) -- built from the
    device selection with one copy (for callers that want the lists; APCalculator does not go through them)."""
    det_mask, scores = select_detections(predicted_boxes, sem_cls_probs, objectness_probs, point_cloud, config_dict)
    corners = predicted_boxes.detach().float().cpu().numpy()
    dm = det_mask.cpu().numpy()
    sc = scores.cpu().numpy()
    out = []
    for i in range(dm.shape[0]):
        cur = []
        if config_dict["per_class_proposal"]:
            for ii in range(sc.shape[-1]):
                cur += [(ii, corners[i, j], sc[i, j, ii]) for j in range(dm.shape[1]) if dm[i, j]]
        else:
            for j in range(dm.shape[1]):
                if dm[i, j]:
                    ii = int(np.argmax(sc[i, j]))
                    cur.append((ii, corners[i, j], sc[i, j, ii]))
        out.append(cur)
    return out


def voc_ap(rec, prec, use_07_metric=False):
    """reference utils/eval_det.py:23-55"""
    if use_07_metric:
        ap = 0.0
        for t in np.arange(0.0, 1.1, 0.1):
            p = 0 if np.sum(rec >= t) == 0 else np.max(prec[rec >= t])
            ap = ap + p / 11.0
        return ap
    mrec = np.concatenate(([0.0], rec, [1.0]))
    mpre = np.concatenate(([0.0], prec, [0.0]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]       # the precision envelope
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


class APCalculator(object):
    """Calculating Average Precision (reference utils/ap_calculator.py:1054-1810), on the device.

    By default the calculator sees every scene it is to score: with data parallelism the caller gathers the batches
    first (the reference's `all_gather_dict`).  `world_size > 1` makes it rank-local, for a data-parallel loop that
    feeds each rank only its own 1/W of every step: scenes are numbered as the gathered stream would number them
    (rank r's scene b of a step is scene (scenes before the step on all ranks) + r * B + b), and `compute_metrics()`
    becomes a collective over `group` that exchanges the ranks' detection records and returns the same dict on every
    rank."""

    def __init__(self, dataset_config, ap_iou_thresh=[0.25, 0.5], class2type_map=None, exact_eval=True, args=None,
                 ap_config_dict=None, reset_nms_iou=None, *, rank=0, world_size=1, group=None):
        self.ap_iou_thresh = ap_iou_thresh
        if ap_config_dict is None:
            ap_config_dict = get_ap_config_dict(dataset_config=dataset_config, remove_empty_box=exact_eval)
        self.ap_config_dict = ap_config_dict
        self.class2type_map = class2type_map
        self.args = args
        self.dataset_config = dataset_config
        self.reset_nms_iou = reset_nms_iou
        if not 0 <= rank < world_size:
            raise ValueError(f"rank {rank} outside a world of {world_size}")
        self.rank, self.world_size, self.group = rank, world_size, group
        self.reset()

    def reset(self):
        self._scores = []          # per step: (B, K, C) f32, -inf = no detection
        self._live = []            # per step: (B, K) bool
        self._tp = []              # per step: (T, B, C, K) bool
        self._scene_base = []      # per step: global number of the step's first scene on this rank
        self._gt_count = None      # (C,) int64 ground-truth boxes per class
        # first appearance of every class among the predictions / the ground truth, in the order the reference's
        # dictionaries are filled (utils/eval_det.py:185-207): its group means (mAP_fre = the first four entries ...)
        # are taken over THAT order
        self._first_pred = None
        self._first_gt = None
        self.scan_cnt = 0

    def step_meter(self, outputs, targets):
        if "outputs" in outputs:
            outputs = outputs["outputs"]
        self.step(
            predicted_box_corners=outputs["box_corners"], sem_cls_probs=outputs["sem_cls_prob"],
            objectness_probs=outputs["objectness_prob"], point_cloud=targets["point_clouds"],
            gt_box_corners=targets["gt_box_corners"], gt_box_sem_cls_labels=targets["gt_box_sem_cls_label"],
            gt_box_present=targets["gt_box_present"])

    @torch.no_grad()
    def step(self, predicted_box_corners, sem_cls_probs, objectness_probs, point_cloud, gt_box_corners,
             gt_box_sem_cls_labels, gt_box_present):
        """NMS + thresholds on the predictions, IoU against the ground truth, matching at every IoU threshold --
        all on the device, accumulated for compute_metrics."""
        cfg = dict(self.ap_config_dict)
        if self.reset_nms_iou is not None:
            cfg["nms_iou"] = self.reset_nms_iou
        det_mask, scores = select_detections(predicted_box_corners, sem_cls_probs, objectness_probs, point_cloud, cfg)
        ncls = scores.shape[-1]
        present = gt_box_present.to(scores.device) > 0
        gcls = gt_box_sem_cls_labels.to(scores.device).long()
        iou = box3d_iou(predicted_box_corners, gt_box_corners.to(scores.device))
        tps = torch.stack([eval_match(iou, scores, det_mask, gcls, present, t) for t in self.ap_iou_thresh])
        self._scores.append(scores)
        self._live.append(det_mask)
        self._tp.append(tps)
        # ground-truth boxes per class (labels outside [0, C) form classes of their own in the reference; the
        # datasets never produce them)
        cnt = torch.zeros(ncls, dtype=torch.int64, device=scores.device)
        cnt.scatter_add_(0, gcls.clamp(0, ncls - 1)[present], torch.ones_like(gcls[present]))
        self._gt_count = cnt if self._gt_count is None else self._gt_count + cnt
        # insertion order of the classes: predictions are listed scene by scene -- class-major for per-class
        # proposals, box by box otherwise -- then the ground truth scene by scene, box by box
        b, k = det_mask.shape
        big = torch.iinfo(torch.int64).max
        base = self.scan_cnt + self.rank * b
        self._scene_base.append(base)
        scene = (base + torch.arange(b, device=scores.device)).view(b, 1, 1)
        is_det = det_mask.unsqueeze(-1) & torch.isfinite(scores)                       # (B, K, C)
        if cfg["per_class_proposal"]:
            pos = (scene * ncls + torch.arange(ncls, device=scores.device).view(1, 1, ncls)) * k \
                + torch.arange(k, device=scores.device).view(1, k, 1)
        else:
            pos = (scene * k + torch.arange(k, device=scores.device).view(1, k, 1)).expand(b, k, ncls)
        first_pred = torch.where(is_det, pos.expand(b, k, ncls), torch.full_like(pos.expand(b, k, ncls), big)).amin(dim=(0, 1))
        g = gcls.shape[1]
        gpos = (base + torch.arange(b, device=scores.device)).view(b, 1) * g + torch.arange(g, device=scores.device)
        first_gt = torch.full((ncls,), big, dtype=torch.int64, device=scores.device)
        first_gt.scatter_reduce_(0, gcls.clamp(0, ncls - 1)[present], gpos[present], reduce="amin")
        self._first_pred = first_pred if self._first_pred is None else torch.minimum(self._first_pred, first_pred)
        self._first_gt = first_gt if self._first_gt is None else torch.minimum(self._first_gt, first_gt)
        self.scan_cnt += self.world_size * b

    # ------------------------------------------------------------------ metrics
    def rank_state(self) -> RankState:
        """This calculator's accumulation as detection records and per-class totals (nothing gathered)."""
        if not self._scores:
            return RankState(None, None, None, None, [])
        rec = eval_records(self._scores, self._live, self._tp, self._scene_base)
        return RankState(rec, self._gt_count, self._first_pred, self._first_gt, [s.shape[0] for s in self._scores])

    def _all_rank_state(self, mine: RankState) -> RankState:
        """The collective behind a rank-local compute_metrics(): every rank ends with the merged state."""
        import torch.distributed as dist

        w, grp = self.world_size, self.group
        # gloo exchanges host tensors, NCCL device tensors; the merged state is reduced on this rank's device
        dev = torch.device("cpu") if dist.get_backend(grp) == "gloo" else torch.device("cuda", torch.cuda.current_device())

        def gather(t):
            parts = [torch.empty_like(t) for _ in range(w)]
            dist.all_gather(parts, t, group=grp)
            return parts

        nsteps = [int(x) for x in gather(torch.tensor([len(mine.batch_sizes)], dtype=torch.int64, device=dev))]
        if len(set(nsteps)) != 1:
            raise ValueError(f"data-parallel evaluation needs the same number of steps on every rank, got {nsteps}")
        if nsteps[0] == 0:
            return mine
        sizes = gather(torch.tensor(mine.batch_sizes, dtype=torch.int64, device=dev))
        _check_batch_sizes([s.tolist() for s in sizes])
        home = mine.gt_count.device
        counts = [int(x) for x in gather(torch.tensor([len(mine.records)], dtype=torch.int64, device=dev))]
        packed = torch.zeros((max(counts), 5), dtype=torch.int32, device=dev)
        packed[:counts[dist.get_rank(grp)]] = pack_records(mine.records).to(dev)
        records = merge_records([unpack_records(p[:n].to(home)) for p, n in zip(gather(packed), counts)])
        totals = []
        for t, op in ((mine.gt_count, dist.ReduceOp.SUM), (mine.first_pred, dist.ReduceOp.MIN),
                      (mine.first_gt, dist.ReduceOp.MIN)):
            t = t.to(dev, copy=True)
            dist.all_reduce(t, op=op, group=grp)
            totals.append(t.to(home))
        return RankState(records, *totals, list(mine.batch_sizes))

    def _class_order(self, classes, first_pred, first_gt):
        """classes in the order the reference's result dictionaries hold them: those that occur among the predictions
        by first occurrence, then the ground-truth-only ones by first occurrence."""
        fp, fg = first_pred.cpu().numpy(), first_gt.cpu().numpy()
        big = np.iinfo(np.int64).max
        return sorted(classes, key=lambda c: (0, fp[c]) if fp[c] < big else (1, fg[c]))

    def compute_metrics(self):
        """Same dict as the reference (:1531-1703): per IoU threshold the per-class AP / Prec / Recall and the
        frequency-group means.  In rank-local mode a collective: every rank must call it, and every rank gets the
        metrics of all ranks' scenes."""
        state = self.rank_state()
        if self.world_size > 1:
            state = self._all_rank_state(state)
        return self.metrics_from_state(state)

    def metrics_from_state(self, state: RankState):
        """compute_metrics() on an accumulated state (`rank_state()`, or `merge_rank_states` of several)."""
        nthr = len(self.ap_iou_thresh)
        if state.gt_count is None:
            classes, ap, last_prec, last_rec, nrec = [], None, None, None, None
        else:
            ncls = state.gt_count.shape[0]
            ap, last_prec, last_rec, counts, _ = eval_ap(sort_records(state.records), ncls, nthr, state.gt_count)
            ap, last_prec, last_rec, nrec, npos = (x.cpu().numpy() for x in (ap, last_prec, last_rec, counts,
                                                                              state.gt_count))
            # the reference only evaluates classes that occur in predictions or ground truth
            classes = [c for c in range(ncls) if nrec[c] > 0 or npos[c] > 0]
        ordered = self._class_order(classes, state.first_pred, state.first_gt) if classes else []
        name = lambda key: self.class2type_map[key] if self.class2type_map else str(key)  # noqa: E731
        overall_ret = OrderedDict()
        for ti, thresh in enumerate(self.ap_iou_thresh):
            ret_dict = OrderedDict()
            for key in classes:
                ret_dict["%s Average Precision" % name(key)] = np.float64(ap[ti, key])
            ap_vals = np.array([ap[ti, key] for key in ordered], dtype=np.float32)
            ap_vals[np.isnan(ap_vals)] = 0
            scannet = (getattr(self.args, "dataset_name", "") or "").find("scannet") != -1 and ap_vals.shape[0] >= 21

            def groups(prefix, vals):
                vals = np.asarray(vals, dtype=np.float64)
                if vals.shape[0] > 2:
                    if not scannet:
                        ret_dict[prefix + "_fre"] = vals[:4].mean()
                        ret_dict[prefix + "_common"] = vals[4:10].mean()
                        ret_dict[prefix + "_base"] = vals[:10].mean()
                        ret_dict[prefix + "_novel"] = vals[10:].mean()
                    else:
                        seen, novel = self.dataset_config.seen_idx_list, self.dataset_config.novel_idx_list
                        ret_dict[prefix + "_fre"] = vals[seen].mean()
                        ret_dict[prefix + "_common"] = vals[seen].mean()
                        ret_dict[prefix + "_base"] = vals[seen].mean()
                        ret_dict[prefix + "_novel"] = vals[novel].mean()

            ret_dict["mAP"] = ap_vals.mean() if ap_vals.size else 0.0
            groups("mAP", ap_vals)
            # per-class entries are emitted by sorted key (:1605-1623), so the LISTS behind the group means are sorted;
            # a class with ground truth but no detection has an empty curve, whose last value the reference reads as 0
            prec_list, rec_list = [], []
            for key in classes:
                last = np.float64(last_prec[ti, key]) if nrec[key] else 0
                ret_dict["%s Prec" % name(key)] = last
                prec_list.append(last)
            for key in classes:
                last = np.float64(last_rec[ti, key]) if nrec[key] else 0
                ret_dict["%s Recall" % name(key)] = last
                rec_list.append(last)
            groups("Prec", prec_list)
            ret_dict["Prec"] = np.mean(prec_list) if prec_list else 0.0
            groups("AR", rec_list)
            ret_dict["AR"] = np.mean(rec_list) if rec_list else 0.0
            overall_ret[thresh] = ret_dict
        return overall_ret

    def __str__(self):
        return self.metrics_to_str(self.compute_metrics())

    def metrics_to_str(self, overall_ret, per_class=True):
        """reference :1709-1793 (same lines, same order)"""
        m_strs, ar_strs, p_strs, per_cls = [], [], [], []
        for t in self.ap_iou_thresh:
            r = overall_ret[t]
            m_strs.append(f"mAP{t:.2f}: {r['mAP'] * 100:.2f}\n")
            if "mAP_fre" in r:
                for g in ("fre", "common", "base"):
                    m_strs.append(f"mAP_{g}{t:.2f}: {r['mAP_' + g] * 100:.2f}\n")
                m_strs.append(f"mAP_novel{t:.2f}: {r['mAP_novel'] * 100:.2f}\n\n")
            ar_strs.append(f"AR{t:.2f}: {r['AR'] * 100:.2f}\n")
            if "AR_fre" in r:
                for g in ("fre", "common", "base"):
                    ar_strs.append(f"AR_{g}{t:.2f}: {r['AR_' + g] * 100:.2f}\n")
                ar_strs.append(f"AR_novel{t:.2f}: {r['AR_novel'] * 100:.2f}\n\n")
            p_strs.append(f"Prec{t:.2f}: {r['Prec'] * 100:.2f}\n")
            if "Prec_fre" in r:
                for g in ("fre", "common", "base"):
                    p_strs.append(f"Prec_{g}{t:.2f}: {r['Prec_' + g] * 100:.2f}\n")
                p_strs.append(f"Prec_novel{t:.2f}: {r['Prec_novel'] * 100:.2f}\n\n")
            if per_class:
                per_cls.append("-" * 5)
                per_cls.append(f"IOU Thresh={t}")
                for x in list(r.keys()):
                    if x in ("mAP", "AR") or x[-3:] == "fre" or x[-6:] == "common" or x[-4:] == "base" or x[-5:] == "novel":
                        continue
                    per_cls.append(f"{x}: {r[x] * 100:.2f}")
        s = "".join(m_strs) + "\n" + "".join(ar_strs) + "\n" + "".join(p_strs) + "\n"
        if per_class:
            s += "\n" + "\n".join(per_cls)
        return s

    def metrics_to_dict(self, overall_ret):
        d = {}
        for t in self.ap_iou_thresh:
            d[f"mAP_{t}"] = overall_ret[t]["mAP"] * 100
            d[f"AR_{t}"] = overall_ret[t]["AR"] * 100
        return d
