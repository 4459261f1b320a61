/*
 * coda_image.h -- C-ABI of the image-side kernel of the CLIP alignment branch.
 */
#ifndef CODA_IMAGE_H
#define CODA_IMAGE_H

#ifdef __cplusplus
extern "C" {
#endif

/*
 * Batched "crop the box, paste it centred on a white square, bicubic-resize the
 * square to res x res, scale to [0,1], normalise" for every selected box of
 * every scene in one launch.
 *   replaces the per-box Python loop of get_predicted_box_clip_embedding
 *   (models/model_3detr.py:1011-1078: img[ymin:ymax, xmin:xmax] -> 255-filled
 *   max_edge^2 canvas -> torchvision Resize(res, BICUBIC) on the uint8 tensor) and
 *   preprocess_for_tensor (CLIP/clip/clip.py:95-101: /255, Normalize(mean, std)).
 *   Resize semantics are torchvision's for a uint8 CUDA tensor: antialiased
 *   bicubic in fp32 (ATen upsample_bicubic2d_aa: cubic a = -0.5, support
 *   2 * max(scale, 1), normalised weights), clamp to [0, 255], round half to
 *   even, as uint8 would hold it.
 *
 *   images   (nimg, h, w, 3) uint8 (HWC, as the dataloader collates them)
 *   scene    (ncrops) int32   image index of each crop
 *   boxes    (ncrops, 4) int32  xmin, ymin, xmax, ymax in pixels (already clipped to the image)
 *   valid    (ncrops) uint8   0 -> the crop is written as zeros
 *   mean/std (3) host floats
 *   out      fp16 if out_half else fp32;  patch == 0: (ncrops, 3, res, res);  patch == ps > 0 (res % ps == 0):
 *            patch-major (ncrops, res / ps, res / ps, 3, ps, ps) -- row (crop, gy, gx) of this buffer is the unfolded
 *            ps x ps patch the ViT's patch-embedding GEMM reads (CLIP/clip/model.py:612-625 conv1 with
 *            kernel = stride = ps), so no unfold copy follows
 *   workspace  coda_crop_resize_workspace_bytes(nimg, h, w) bytes: an RGBX copy of the images (one 32-bit load per
 *            filter tap instead of three byte loads)
 *   tile_rows  0 = automatic; output rows per CTA (tuning / tests)
 *
 * The resize is evaluated in its separable form -- a CTA resamples the source rows of its output rows horizontally
 * into shared memory, then vertically -- with the sums in the order of the direct double loop (same bits).
 */
long long coda_crop_resize_workspace_bytes(int nimg, int h, int w);
int coda_crop_resize_normalize_ex(int nimg, int h, int w, int ncrops, int res,
                                  const unsigned char *images, const int *scene,
                                  const int *boxes, const unsigned char *valid,
                                  const float *mean, const float *std, int out_half,
                                  int patch, int tile_rows, void *workspace, void *out,
                                  void *stream);

/*
 * Test-time classification of predicted boxes by their CLIP crops (the baseline head's `if_real_test` path;
 * replaces the normalise / matmul / softmax / index-put of reference models/model_3detr.py:3056-3064).
 *   feats    (n, d) fp32    CLIP image features of the n compacted crops
 *   text     (c, d) fp32    L2-normalised text features of the c class prompts
 *   scale    (1) fp32, device   the logit scale (read on the device: no host synchronisation)
 *   row_map  (rows) int32   row of `feats` for each (scene, query) row; -1 (or anything outside [0, n)) = skipped
 *   prob     (rows, c) fp32  usable rows: softmax(scale * (f / |f|) . text^T); skipped rows: exact zeros
 *   logits   (rows, c) fp32  written as zeros (the reference leaves sem_cls_logits at zero), may be NULL
 * The norm, the dot products and the max-subtracted softmax are evaluated in fp64 from the fp32 operands and
 * rounded once to fp32, in a fixed order: the result is the same bits on every run.  Nothing outside prob and
 * logits is written; no allocation.  d must be 512 (CODA_EINVAL otherwise); c from 1 to 28000.
 */
int coda_clip_classify(long long rows, int n, int c, int d, const float *feats, const float *text,
                       const float *scale, const int *row_map, float *prob, float *logits, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CODA_IMAGE_H */
