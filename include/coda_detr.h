/*
 * coda_detr.h -- C-ABI of the warp-primitive kernels of the 3DETR encoder /
 * decoder, box geometry and matcher (everything on the training-step path that
 * is not a dense contraction; the tensor-core attention is in coda_attention.h).
 *
 * Conventions as in coda_pointnet2.h: raw device pointers, dense row-major fp32
 * unless stated, `void *stream` is a cudaStream_t, int status (0 = ok).
 * The reference has no native code for these ops -- it reaches them through
 * PyTorch (SURVEY.md section 2b); each entry cites the Python it replaces.
 */
#ifndef CODA_DETR_H
#define CODA_DETR_H

#ifdef __cplusplus
extern "C" {
#endif

/*
 * LayerNorm over the last dimension, one warp per row.
 *   replaces nn.LayerNorm in TransformerEncoderLayer / TransformerDecoderLayer
 *   (models/transformer.py:461-479, :556-580; NORM_DICT["ln"], models/helpers.py:27-32)
 *   x, y (rows, c); gamma, beta (c); mean, rstd (rows) saved for backward.
 *   c must be a multiple of 128 and <= 1024.
 */
int coda_layer_norm_fwd(long long rows, int c, float eps, const float *x,
                        const float *gamma, const float *beta, float *y,
                        float *mean, float *rstd, void *stream);
/*
 * The same with the transformer layer's neighbours folded in (models/transformer.py:556-580: `tgt2 = self.norm1(tgt);
 * q = k = self.with_pos_embed(tgt2, query_pos)`; models/transformer.py:97-143: the decoder's `self.norm(output)` of
 * every layer stacked, which models/model_3detr.py:1634-1650 then permutes to (layer, batch, query)):
 *   y      may be NULL; row r of y is written at  r * c  floats when y_inner == 0, else at
 *          (r / y_inner) * y_so + (r % y_inner) * y_si  (multiples of 4) -- a row permutation / a slice of a larger
 *          buffer without a copy
 *   y_pos  (rows, c) = y + pos  when pos != NULL (both or neither)
 */
int coda_layer_norm_fwd_ex(long long rows, int c, float eps, const float *x,
                           const float *gamma, const float *beta, float *y, int y_inner,
                           long long y_so, long long y_si, const float *pos, float *y_pos,
                           float *mean, float *rstd, void *stream);
/*
 * Forward-only variant for fp16 activations: x, y are IEEE half (rows, c); gamma,
 * beta fp32; statistics in fp32 and one rounding to half at the end.
 *   replaces the fp32-upcasting LayerNorm of the CLIP towers
 *   (CLIP/clip/model.py:254-260: `super().forward(x.type(torch.float32)).type(orig_type)`)
 */
int coda_layer_norm_fwd_half(long long rows, int c, float eps, const void *x,
                             const float *gamma, const float *beta, void *y,
                             void *stream);
/*
 *   dx (rows, c) may alias dy.  dgamma / dbeta (c) are fully written.
 *   `partial` is caller-provided scratch of coda_layer_norm_bwd_scratch(rows, c)
 *   floats (block partial sums, reduced deterministically).
 */
long long coda_layer_norm_bwd_scratch(long long rows, int c);
int coda_layer_norm_bwd(long long rows, int c, const float *dy, const float *x,
                        const float *gamma, const float *mean, const float *rstd,
                        float *dx, float *dgamma, float *dbeta, float *partial,
                        void *stream);
/*
 * Backward of coda_layer_norm_fwd_ex and of the residual connection around the norm, in one pass:
 *   d  = dy (row-mapped like y above) + dy2 (optional (rows, c): the gradient that arrived through y_pos)
 *   dx = LayerNormBackward(d) + add   (add optional (rows, c): the gradient of `tgt` through the branch that
 *        by-passes the norm -- autograd would otherwise run a separate `grad_a + grad_b` kernel per norm)
 *   dgamma / dbeta from d.  dx may alias dy, dy2 or add.
 */
int coda_layer_norm_bwd_ex(long long rows, int c, const float *dy, int dy_inner, long long dy_so,
                           long long dy_si, const float *dy2, const float *add, const float *x,
                           const float *gamma, const float *mean, const float *rstd,
                           float *dx, float *dgamma, float *dbeta, float *partial,
                           void *stream);

/*
 * Row softmax / log-softmax over the last dimension (any c >= 1), one warp per row.
 *   replaces torch.nn.functional.softmax call sites on the path
 *   (models/model_3detr.py:99 objectness, :1160 weak labels; criterion.py cross-entropy)
 */
int coda_softmax_rows(long long rows, int c, int log_softmax, const float *x,
                      float *y, void *stream);

/*
 * Fourier positional encoding, fused: shift/scale to the scene range, * 2 pi,
 * 3 x d_out projection, sin | cos, channel-major store.
 *   replaces PositionEmbeddingCoordsSine.get_fourier_embeddings
 *   (models/position_embedding.py:89-118) + shift_scale_points (utils/pc_util.py:38-66)
 *   xyz (b, n, 3); range_min/range_max (b, 3) or NULL when normalize == 0;
 *   gauss_b (3, ldb) row-major, first d_out columns used; out (b, 2*d_out, n).
 */
int coda_fourier_pos_embed(int b, int n, int d_out, int ldb, int normalize,
                           const float *xyz, const float *range_min,
                           const float *range_max, const float *gauss_b,
                           float *out, void *stream);

/*
 * Generalised 3-D IoU between predicted and ground-truth boxes, one thread per
 * (scene, proposal, gt) triple, including the rotated-rectangle intersection
 * (Sutherland-Hodgman clip of the two ground-plane rectangles).
 *   replaces generalized_box3d_iou (utils/box_util.py:855-875) and what it calls:
 *   generalized_box3d_iou_tensor (:655-757), enclosing_box3d_vol (:604-652),
 *   box3d_vol_tensor (:581-601), polygon_clip_unnest (:540-578) -- and the
 *   Cython copy utils/box_intersection.pyx:167-199.
 *   corners1 (b, k1, 8, 3), corners2 (b, k2, 8, 3)  (camera frame, up = -Y),
 *   nums_k2 (b) int32 number of real gt boxes per scene (columns >= nums_k2 -> 0),
 *   rotated: 0 = axis-aligned intersection, 1 = polygon clip; if rotated_dev is not NULL
 *     the flag is read from that device int instead (the reference derives it from
 *     torch.any(gt_angles > 0).item(), criterion.py:1111 -- a host sync this avoids);
 *   rot_k2_limit: polygon clip only for gt index < limit, others get area 0
 *     (pass 4 to reproduce the compiled-Cython reference, whose loop bound is
 *      rect2.shape[2] == 4, box_intersection.pyx:181; pass k2 for the intended /
 *      TorchScript behaviour).
 *   gious (b, k1, k2).
 */
int coda_giou3d(int b, int k1, int k2, int rotated, const int *rotated_dev,
                int rot_k2_limit, const float *corners1, const float *corners2,
                const int *nums_k2, float *gious, void *stream);

/*
 * Hungarian matching of proposals to ground truth, one CTA per scene.
 *   replaces Matcher.forward's per-scene scipy.optimize.linear_sum_assignment
 *   (criterion.py:59-80); cost (b, nprop, ngt) fp32 (final_cost, criterion.py:52-57),
 *   nactual (b) int32.  Solves min sum cost[i, assign(j)] over the first nactual[b]
 *   columns (each gt gets a distinct proposal; nprop >= nactual).
 *   per_prop_gt_inds (b, nprop) int64 (0 where unmatched), proposal_matched_mask
 *   (b, nprop) fp32 in {0, 1}.  Arithmetic in fp64 like scipy.
 */
int coda_hungarian(int b, int nprop, int ngt, const float *cost, const int *nactual,
                   long long *per_prop_gt_inds, float *proposal_matched_mask,
                   void *stream);

/*
 * Stage-2 novel-box discovery, candidate selection (one CTA per scene, no host synchronisation):
 *   replaces models/model_3detr.py:1298-1420 -- the per-box loop building `box2d_thisbatch` / `scores`,
 *   torchvision.ops.nms(box2d, scores, 0.25) (:1348), the cal_iou double loop against the ground truth (:1374-1386,
 *   :868-899) and the `box_save` thresholding (:1402-1420).
 *   boxes2d (b, q, 4) int32 projected boxes, valid (b, q) uint8 (0 = box given up: its NMS box is the dummy
 *   (0, 0, 2, 2) and its score -1, as in the reference), objectness (b, q), pred_corners (b, q, 8, 3),
 *   gt_corners (b, g, 8, 3), gt_present (b, g) in {0, 1}.
 *   A box is a candidate iff it survives the class-agnostic 2-D NMS (IoU > nms_iou suppresses, score order), is
 *   valid, has objectness >= min_objectness (a NaN objectness is not below it) and its axis-aligned 3-D IoU with every
 *   present ground-truth box is <= gt_iou.  The score order is total, like the stable descending sort of
 *   torchvision.ops.nms: NaN above every number, then descending value, ties (NaN with NaN, -0.0 with +0.0) by lower
 *   index.  cand_idx (b, cap) int32: candidate box indices in that order, -1 padded;
 *   cand_count (b, 2) int32: entries written, and the untruncated total (total > written: raise `cap`).
 *   q from 1 to 1024 and cap >= 1 (CODA_EINVAL otherwise).
 */
int coda_novel_candidates(int b, int q, int g, int cap, const int *boxes2d, const unsigned char *valid,
                          const float *objectness, const float *pred_corners, const float *gt_corners,
                          const float *gt_present, float nms_iou, float gt_iou, float min_objectness, int *cand_idx,
                          int *cand_count, void *stream);

/*
 * Predicted 3-D boxes -> integer 2-D boxes in the image + usability flags, one thread per box, fp64.
 *   replaces models/model_3detr.py:912-968 (undo scale / rotation / flips of the point-cloud augmentation), the
 *   dataset's project_3dpoint_to_2dpoint_corners_tensor, the clipping / offset / image-flip bookkeeping (:950-968)
 *   and the per-box checks (:1034-1051).  `camera` picks the dataset's camera model (model_3detr.py:461-466):
 *     CODA_CAMERA_SUNRGBD  datasets/sunrgbd_utils.py:611-635: K (3x3 intrinsics), Rtilt (3x3 tilt);
 *                          p_cam = axis swap of Rtilt^T p, uv = K p_cam.
 *     CODA_CAMERA_SCANNET  datasets/scannet_utils.py:650-690: K (4x4 intrinsic_color), Rtilt (4x4 camera-to-world
 *                          pose); p_cam = inv(pose) [p, 1] (rows 0..2; the inverse by Gauss-Jordan with partial
 *                          pivoting, once per scene, fp64), uv = K[:3, :3] p_cam.
 *   Both: pixel = uv[0:2] / (uv[2] + 1e-32), depth = uv[2].
 *   corners_xyz (b, q, 8, 3) fp32, size_unnorm (b, q, 3) fp32; per scene (fp64, row-major): scale (3), rot (3x3,
 *   applied as p @ rot), flip, zx_flip (NULL = absent), K, Rtilt, img_flip, flip_len; (int64): ori_w, ori_h, x_off,
 *   y_off.  boxes (b, q, 4) int32 [xmin, ymin, xmax, ymax] (truncation, like int(torch.min(.)));
 *   valid (b, q) uint8 = (xmax > xmin) & (ymax > ymin) & (min depth >= 0) & !(max size < 1e-16) (and, ScanNet, a
 *   non-singular pose); extent (b, q, 4) fp64 [umin, vmin, umax, vmax] before truncation, or NULL (not written).
 */
#define CODA_CAMERA_SUNRGBD 0
#define CODA_CAMERA_SCANNET 1
int coda_boxes_in_image(int b, int q, int camera, const float *corners_xyz, const float *size_unnorm,
                        const double *scale, const double *rot, const double *flip, const double *zx_flip,
                        const double *K, const double *Rtilt, const long long *ori_w, const long long *ori_h,
                        const long long *x_off, const long long *y_off, const double *img_flip,
                        const double *flip_len, int *boxes, unsigned char *valid, double *extent, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_DETR_H */
