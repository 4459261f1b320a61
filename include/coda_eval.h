/*
 * coda_eval.h -- C-ABI of the evaluation path (SURVEY.md section 8 row f4): what utils/ap_calculator.py does on the
 * host with numpy / scipy, one box at a time, as batched device kernels.  Conventions as in coda_pointnet2.h: raw
 * device pointers, dense row-major, `void *stream` is a cudaStream_t, int status (0 = ok); no host synchronisation.
 *
 * Box corners are (8, 3) fp32 in the order of utils/box_util.py get_3d_box (:383-407): corners 0-3 the upper face,
 * 4-7 the lower one; edge 0-1 spans w, 1-2 spans l, 0-4 spans h; upright CAMERA frame (x right, y down, z forward).
 */
#ifndef CODA_EVAL_H
#define CODA_EVAL_H

#include "coda_pointnet2.h" /* status codes */

#ifdef __cplusplus
extern "C" {
#endif

/*
 * counts (b, k) int32 = number of points of scene b inside predicted box (b, j).
 *   replaces the `remove_empty_box` loop of parse_predictions (utils/ap_calculator.py:808-835): per box
 *   flip_axis_to_depth + extract_pc_in_box3d (utils/box_util.py:22-31, a scipy Delaunay hull test on the host).
 *   corners_camera (b, k, 8, 3) camera frame; points_depth (b, n, point_stride) fp32 in the upright DEPTH frame
 *   (depth (X, Y, Z) = camera (X, Z, -Y)), only the first three columns are read.  Faces are inclusive: a point on
 *   a face, an edge or a corner of the box is inside.  A box with an edge of length zero -- the all-zero box, a box
 *   of zero height -- has no inside and counts 0.
 */
int coda_points_in_boxes(int b, int k, int n, int point_stride, const float *corners_camera, const float *points_depth,
                         int *counts, void *stream);

/*
 * Greedy 3-D non-maximum suppression per scene on the axis-aligned extents of the corners.
 *   replaces nms_3d_faster / nms_3d_faster_samecls (utils/nms.py:79-162) and the per-scene Python loops that build
 *   their input (utils/ap_calculator.py:868-941).  Candidates are the boxes with valid != 0 whose score is not NaN
 *   (a NaN cannot be ranked; such a box is never kept, whatever `valid` says; -inf and +inf are ordinary scores);
 *   visited from the highest score, among equal scores the higher index first; a later box is dropped when
 *   inter / (vol_i + vol_j - inter) > iou_thresh (old_type: inter / vol_j) and -- if cls is not NULL -- it has the
 *   same class.  keep (b, k) uint8, k <= 2048.
 */
int coda_nms3d(int b, int k, const float *corners, const float *score, const int *cls, const unsigned char *valid,
               float iou_thresh, int old_type, unsigned char *keep, void *stream);

/*
 * ious (b, k1, k2) = 3-D IoU of boxes that are rotated about the up axis: ground-plane polygon clip x height overlap
 *   / (vol1 + vol2 - intersection).   replaces box3d_iou (utils/box_util.py:156-183) called pair by pair from
 *   eval_det_cls (utils/eval_det.py:122-130).
 */
int coda_box3d_iou(int b, int k1, int k2, const float *corners1, const float *corners2, float *ious, void *stream);

/*
 * VOC matching of detections to ground truth, one warp per (scene, class):
 *   tp (b, ncls, k) uint8 = 1 where detection j, scored scores[b, j, c] for class c, is a true positive at
 *   `iou_thresh`: visiting the scene's live detections (det_mask) in descending score order, each looks up the
 *   ground-truth box of class c (gt_cls (b, g) int32, gt_present (b, g) uint8) with the largest iou (b, k, g) and
 *   claims it if that IoU > iou_thresh and it is still unclaimed.   replaces the inner loop of eval_det_cls
 *   (utils/eval_det.py:110-146); the precision / recall curves over the whole dataset follow from (score, tp).
 */
int coda_eval_match(int b, int k, int g, int ncls, const float *iou, const float *scores,
                    const unsigned char *det_mask, const int *gt_cls, const unsigned char *gt_present, float iou_thresh,
                    unsigned char *tp, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_EVAL_H */
