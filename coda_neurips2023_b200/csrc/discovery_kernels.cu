// Stage-2 novel-box discovery on the device (sm_90a): class-agnostic 2-D NMS of the projected boxes, rejection of
// boxes that overlap a ground-truth box in 3-D, objectness threshold, emitted as a fixed-capacity candidate list per
// scene -- so that the step stays free of host synchronisation and CUDA-graph capturable.
//
// Replaces, in get_predicted_box_clip_embedding_nms_iou_save_keep_clip_driven_with_cate_confidence
// (models/model_3detr.py:1298-1420): the per-box Python loop that builds box2d / scores with four .item() syncs per
// box (:1303-1346), torchvision.ops.nms (:1348), the Python double loop over cal_iou (:1374-1386, :868-899) and the
// box_save bookkeeping (:1402-1420).  C-ABI in include/coda_detr.h.
#include <math.h>
#include <stdint.h>

#include "../../include/coda_detr.h"
#include "coda_common.cuh"

using namespace coda;

namespace {

constexpr int MAXQ = 1024;

__global__ void __launch_bounds__(256)
novel_candidates_kernel(int q, int g, int cap, const int *__restrict__ boxes2d, const unsigned char *__restrict__ valid,
                        const float *__restrict__ objectness, const float *__restrict__ pred_corners,
                        const float *__restrict__ gt_corners, const float *__restrict__ gt_present, float nms_iou,
                        float gt_iou, float min_objectness, int *__restrict__ cand_idx, int *__restrict__ cand_count) {
  extern __shared__ unsigned char smem_raw[];
  const int words = (q + 31) / 32;
  float *score = reinterpret_cast<float *>(smem_raw);            // [q]
  float4 *box = reinterpret_cast<float4 *>(score + q);           // [q]  (x1, y1, x2, y2), in score order
  int *order = reinterpret_cast<int *>(box + q);                 // [q]  rank -> box index
  uint32_t *sup = reinterpret_cast<uint32_t *>(order + q);       // [q][words]  suppression bits (row a: later boxes b)
  uint32_t *keep = sup + (size_t)q * words;                      // [words]
  unsigned char *ok = reinterpret_cast<unsigned char *>(keep + words);   // [q] survives gt filter + thresholds
  const int b = blockIdx.x, tid = threadIdx.x;
  const int *bx = boxes2d + (size_t)b * q * 4;
  // scores: objectness, -1 for a box that was given up (degenerate crop / behind the camera / zero size)
  for (int i = tid; i < q; i += blockDim.x) score[i] = valid[(size_t)b * q + i] ? objectness[(size_t)b * q + i] : -1.0f;
  __syncthreads();
  // descending order (ties: lower index first), by counting
  for (int i = tid; i < q; i += blockDim.x) {
    const float s = score[i];
    int r = 0;
    for (int j = 0; j < q; ++j) {
      const float t = score[j];
      r += (t > s) || (t == s && j < i);
    }
    order[r] = i;
  }
  __syncthreads();
  for (int a = tid; a < q; a += blockDim.x) {
    const int i = order[a];
    // a given-up box enters the NMS as the dummy (0, 0, 2, 2) like in the reference (:1305-1311)
    box[a] = valid[(size_t)b * q + i] ? make_float4((float)bx[4 * i], (float)bx[4 * i + 1], (float)bx[4 * i + 2], (float)bx[4 * i + 3])
                                      : make_float4(0.f, 0.f, 2.f, 2.f);
  }
  __syncthreads();
  // suppression matrix (torchvision nms: inter / (Sa + Sb - inter) > thr)
  for (int a = tid; a < q; a += blockDim.x) {
    const float4 A = box[a];
    const float sa = (A.z - A.x) * (A.w - A.y);
    for (int w = 0; w < words; ++w) {
      uint32_t bits = 0;
      for (int k = 0; k < 32; ++k) {
        const int c = w * 32 + k;
        if (c > a && c < q) {
          const float4 B = box[c];
          const float iw = fmaxf(fminf(A.z, B.z) - fmaxf(A.x, B.x), 0.f), ih = fmaxf(fminf(A.w, B.w) - fmaxf(A.y, B.y), 0.f);
          const float inter = iw * ih, sb = (B.z - B.x) * (B.w - B.y);
          if (inter / (sa + sb - inter) > nms_iou) bits |= 1u << k;
        }
      }
      sup[(size_t)a * words + w] = bits;
    }
  }
  __syncthreads();
  if (tid < 32) {
    // greedy sweep in score order, one warp: lane w owns word w of the removed mask (words <= 32)
    uint32_t removed = 0, kept = 0;
    for (int a = 0; a < q; ++a) {
      const uint32_t rw = __shfl_sync(0xffffffffu, removed, a >> 5);
      const bool alive = !((rw >> (a & 31)) & 1u);
      if (alive) {
        if (tid < words) removed |= sup[(size_t)a * words + tid];
        if (tid == (a >> 5)) kept |= 1u << (a & 31);
      }
    }
    if (tid < words) keep[tid] = kept;
  }
  __syncthreads();
  // 3-D axis-aligned IoU of each kept box against every present ground-truth box (cal_iou, :868-899)
  for (int a = tid; a < q; a += blockDim.x) {
    const int i = order[a];
    bool good = (keep[a >> 5] >> (a & 31)) & 1u;
    good = good && valid[(size_t)b * q + i] && !(score[i] < min_objectness);
    if (good) {
      const float *pc = pred_corners + ((size_t)b * q + i) * 24;
      float lo[3] = {pc[0], pc[1], pc[2]}, hi[3] = {pc[0], pc[1], pc[2]};
      for (int c = 1; c < 8; ++c)
        for (int d = 0; d < 3; ++d) { lo[d] = fminf(lo[d], pc[c * 3 + d]); hi[d] = fmaxf(hi[d], pc[c * 3 + d]); }
      const float v1 = (hi[0] - lo[0]) * (hi[1] - lo[1]) * (hi[2] - lo[2]);
      for (int k = 0; k < g && good; ++k) {
        if (gt_present[(size_t)b * g + k] == 0.f) continue;
        const float *gc = gt_corners + ((size_t)b * g + k) * 24;
        float glo[3] = {gc[0], gc[1], gc[2]}, ghi[3] = {gc[0], gc[1], gc[2]};
        for (int c = 1; c < 8; ++c)
          for (int d = 0; d < 3; ++d) { glo[d] = fminf(glo[d], gc[c * 3 + d]); ghi[d] = fmaxf(ghi[d], gc[c * 3 + d]); }
        float inter = 1.f;
        for (int d = 0; d < 3; ++d) inter *= fmaxf(fminf(hi[d], ghi[d]) - fmaxf(lo[d], glo[d]), 0.f);
        const float v2 = (ghi[0] - glo[0]) * (ghi[1] - glo[1]) * (ghi[2] - glo[2]);
        if (inter / (v1 + v2 - inter) > gt_iou) good = false;
      }
    }
    ok[a] = good ? 1 : 0;
  }
  __syncthreads();
  if (tid == 0) {
    int n = 0, total = 0;
    for (int a = 0; a < q; ++a) {
      if (ok[a]) {
        if (n < cap) cand_idx[(size_t)b * cap + n++] = order[a];
        ++total;
      }
    }
    for (int k = n; k < cap; ++k) cand_idx[(size_t)b * cap + k] = -1;
    cand_count[2 * b] = n;
    cand_count[2 * b + 1] = total;     // > n: the capacity truncated the list
  }
}

}  // namespace

extern "C" {

int coda_novel_candidates(int b, int q, int g, int cap, const int *boxes2d, const unsigned char *valid,
                          const float *objectness, const float *pred_corners, const float *gt_corners,
                          const float *gt_present, float nms_iou, float gt_iou, float min_objectness, int *cand_idx,
                          int *cand_count, void *stream) {
  if (b < 0 || q < 1 || q > MAXQ || g < 0 || cap < 1) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!boxes2d || !valid || !objectness || !pred_corners || !cand_idx || !cand_count || (g > 0 && (!gt_corners || !gt_present)))
    return CODA_EINVAL;
  const int words = (q + 31) / 32;
  const size_t smem = (size_t)q * (4 + 16 + 4) + (size_t)q * words * 4 + (size_t)words * 4 + q + 16;
  if (smem > 200 * 1024) return CODA_ETOOLARGE;
  cudaError_t e = cudaFuncSetAttribute(novel_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  novel_candidates_kernel<<<b, 256, smem, (cudaStream_t)stream>>>(q, g, cap, boxes2d, valid, objectness, pred_corners,
                                                                gt_corners, gt_present, nms_iou, gt_iou, min_objectness,
                                                                cand_idx, cand_count);
  return launch_status();
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Predicted 3-D boxes -> 2-D boxes in the image (one thread per box, fp64 like the reference):
//   undo the point-cloud augmentation (scale, rotation, flips), rotate into the camera frame (Rtilt^T), project with
//   K, clip to the original image, add the crop offsets, undo the image flip, then the integer bounding box of the
//   eight projected corners (truncation of non-negative values, as `int(torch.min(.))`) and the usability flag.
// Replaces models/model_3detr.py:912-968 + datasets/sunrgbd_utils.py:611-635 (project_3dpoint_to_2dpoint_corners_tensor)
// + the per-box checks of :1034-1051 -- in the reference a chain of fp64 tensor ops plus four .item() syncs per box.
namespace {

__global__ void __launch_bounds__(128)
boxes_in_image_kernel(int b, int q, const float *__restrict__ corners, const float *__restrict__ size,
                      const double *__restrict__ scale, const double *__restrict__ rot, const double *__restrict__ flip,
                      const double *__restrict__ zx_flip, const double *__restrict__ Kmat,
                      const double *__restrict__ Rtilt, const long long *__restrict__ ori_w,
                      const long long *__restrict__ ori_h, const long long *__restrict__ x_off,
                      const long long *__restrict__ y_off, const double *__restrict__ img_flip,
                      const double *__restrict__ flip_len, int *__restrict__ boxes, unsigned char *__restrict__ valid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b * q) return;
  const int s = i / q;
  const double *R = rot + s * 9, *T = Rtilt + s * 9, *K = Kmat + s * 9, *sc = scale + s * 3;
  const double fx = flip[s], zx = zx_flip ? zx_flip[s] : 1.0;
  const double wmax = (double)(ori_w[s] - 1), hmax = (double)(ori_h[s] - 1);
  const double yo = (double)y_off[s], xo = (double)x_off[s], fl = img_flip[s], flen = flip_len[s];
  double umin = 1e300, vmin = 1e300, umax = -1e300, vmax = -1e300, dmin = 1e300;
  const float *c = corners + (size_t)i * 24;
  for (int k = 0; k < 8; ++k) {
    const double p0 = (double)c[k * 3] * sc[0], p1 = (double)c[k * 3 + 1] * sc[1], p2 = (double)c[k * 3 + 2] * sc[2];
    double r0 = p0 * R[0] + p1 * R[3] + p2 * R[6];      // row vector times rot_array
    double r1 = p0 * R[1] + p1 * R[4] + p2 * R[7];
    const double r2 = p0 * R[2] + p1 * R[5] + p2 * R[8];
    r1 *= zx;
    r0 *= fx;
    const double t0 = T[0] * r0 + T[3] * r1 + T[6] * r2;   // Rtilt^T p
    const double t1 = T[1] * r0 + T[4] * r1 + T[7] * r2;
    const double t2 = T[2] * r0 + T[5] * r1 + T[8] * r2;
    const double c0 = t0, c1 = -t2, c2 = t1;               // depth -> camera axes
    const double u3 = c0 * K[0] + c1 * K[1] + c2 * K[2];
    const double v3 = c0 * K[3] + c1 * K[4] + c2 * K[5];
    const double d = c0 * K[6] + c1 * K[7] + c2 * K[8];
    double u = u3 / (d + 1e-32), v = v3 / (d + 1e-32);
    u = fmin(fmax(u, 0.0), wmax) + yo;
    v = fmin(fmax(v, 0.0), hmax) + xo;
    u = u * fl + (1.0 - fl) * (flen - 1.0 - u);
    umin = fmin(umin, u); umax = fmax(umax, u);
    vmin = fmin(vmin, v); vmax = fmax(vmax, v);
    dmin = fmin(dmin, d);
  }
  const int xmin = (int)umin, ymin = (int)vmin, xmax = (int)umax, ymax = (int)vmax;
  boxes[4 * i] = xmin; boxes[4 * i + 1] = ymin; boxes[4 * i + 2] = xmax; boxes[4 * i + 3] = ymax;
  const float smax = fmaxf(size[3 * i], fmaxf(size[3 * i + 1], size[3 * i + 2]));
  valid[i] = ((xmax - xmin) > 0 && (ymax - ymin) > 0 && dmin >= 0.0 && !(smax < 1e-16f)) ? 1 : 0;
}

}  // namespace

extern "C" int coda_boxes_in_image(int b, int q, const float *corners_xyz, const float *size_unnorm,
                                   const double *scale, const double *rot, const double *flip, const double *zx_flip,
                                   const double *K, const double *Rtilt, const long long *ori_w, const long long *ori_h,
                                   const long long *x_off, const long long *y_off, const double *img_flip,
                                   const double *flip_len, int *boxes, unsigned char *valid, void *stream) {
  if (b < 0 || q < 0) return CODA_EINVAL;
  if (b == 0 || q == 0) return CODA_OK;
  if (!corners_xyz || !size_unnorm || !scale || !rot || !flip || !K || !Rtilt || !ori_w || !ori_h || !x_off || !y_off ||
      !img_flip || !flip_len || !boxes || !valid)
    return CODA_EINVAL;
  boxes_in_image_kernel<<<(b * q + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      b, q, corners_xyz, size_unnorm, scale, rot, flip, zx_flip, K, Rtilt, ori_w, ori_h, x_off, y_off, img_flip, flip_len,
      boxes, valid);
  return launch_status();
}
