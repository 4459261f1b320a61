// Evaluation path on the device (sm_90a): what the reference's APCalculator does box by box on the host with numpy /
// scipy (utils/ap_calculator.py, utils/nms.py, utils/eval_det.py, utils/box_util.py) as four batched kernels.
//
//   points_in_boxes   -- "remove_empty_box": how many points of the scene lie inside each predicted box
//                        (ap_calculator.py:808-835: a scipy Delaunay hull test per box; here three dot products
//                        against the box's edge frame, one thread per box, the scene streamed through shared memory)
//   nms3d             -- greedy 3-D NMS on the axis-aligned extents, optionally only between boxes of the same class
//                        (utils/nms.py:79-162, called per scene at ap_calculator.py:875-941)
//   box3d_iou         -- IoU of every (detection, ground-truth) pair incl. the rotated ground-plane polygon clip
//                        (utils/box_util.py:156-183, called pair by pair from utils/eval_det.py:122-130)
//   eval_match        -- VOC matching per (scene, class): detections in descending score order claim the ground-truth
//                        box of their class they overlap most (utils/eval_det.py:110-146)
// Nothing here synchronises with the host; a whole evaluation step is five launches.  C-ABI in include/coda_eval.h.
#include <math.h>
#include <stdint.h>

#include "../../include/coda_eval.h"
#include "box_geometry.cuh"
#include "coda_common.cuh"

using namespace coda;

namespace {

// ------------------------------------------------------------------ points inside boxes
// corners (b, k, 8, 3) in the upright CAMERA frame (x right, y down, z forward) in the order of get_3d_box
// (utils/box_util.py:383-407: 0-1 spans the w edge, 0-3 the l edge, 0-4 the h edge); points (b, n, >=3) in the
// upright DEPTH frame.  depth (X, Y, Z) = camera (X, Z, -Y)  (ap_calculator.py:24-28 flip_axis_to_depth).
constexpr int PIB_TILE = 1024;

__global__ void __launch_bounds__(128)
points_in_boxes_kernel(int k, int n, int pstride, const float *__restrict__ corners, const float *__restrict__ points,
                       int *__restrict__ counts) {
  __shared__ float3 pts[PIB_TILE];
  const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = j < k;
  float3 o = make_float3(0.f, 0.f, 0.f), u = o, v = o, w = o;
  float uu = 0.f, vv = 0.f, ww = 0.f;
  if (live) {
    const float *c = corners + ((size_t)b * k + j) * 24;
    // camera -> depth: (x, y, z) -> (x, z, -y)
    auto dep = [&](int q) { return make_float3(c[q * 3], c[q * 3 + 2], -c[q * 3 + 1]); };
    o = dep(0);
    const float3 c1 = dep(1), c3 = dep(3), c4 = dep(4);
    u = make_float3(c1.x - o.x, c1.y - o.y, c1.z - o.z);
    v = make_float3(c3.x - o.x, c3.y - o.y, c3.z - o.z);
    w = make_float3(c4.x - o.x, c4.y - o.y, c4.z - o.z);
    uu = u.x * u.x + u.y * u.y + u.z * u.z;
    vv = v.x * v.x + v.y * v.y + v.z * v.z;
    ww = w.x * w.x + w.y * w.y + w.z * w.z;
  }
  // inclusive faces, with the slack a hull test in double precision has around an fp32 box
  const float eu = 1e-6f * uu, ev = 1e-6f * vv, ew = 1e-6f * ww;
  // a box with an edge of length zero (the all-zero padding box among them) has no inside: without this every
  // comparison below reads 0 >= -0 && 0 <= 0 along that edge and the flat box would collect the points of its plane
  const bool solid = live && uu > 0.f && vv > 0.f && ww > 0.f;
  int cnt = 0;
  for (int p0 = 0; p0 < n; p0 += PIB_TILE) {
    const int m = min(PIB_TILE, n - p0);
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
      const float *p = points + ((size_t)b * n + p0 + i) * pstride;
      pts[i] = make_float3(p[0], p[1], p[2]);
    }
    __syncthreads();
    if (solid) {
      for (int i = 0; i < m; ++i) {
        const float dx = pts[i].x - o.x, dy = pts[i].y - o.y, dz = pts[i].z - o.z;
        const float a = dx * u.x + dy * u.y + dz * u.z;
        const float bb = dx * v.x + dy * v.y + dz * v.z;
        const float cc = dx * w.x + dy * w.y + dz * w.z;
        cnt += (a >= -eu && a <= uu + eu && bb >= -ev && bb <= vv + ev && cc >= -ew && cc <= ww + ew) ? 1 : 0;
      }
    }
  }
  if (live) counts[(size_t)b * k + j] = cnt;
}

// ------------------------------------------------------------------ 3-D NMS
// One CTA per scene.  Boxes enter by their axis-aligned extents in the frame they are given in (the reference feeds
// the camera-frame corners, ap_calculator.py:877-899); candidates = valid boxes whose score is not NaN; greedy from
// the highest score (utils/nms.py:90-116 walks np.argsort(score) from the back: among equal scores the higher index
// goes first).
constexpr int NMS_MAXK = 2048;

__global__ void __launch_bounds__(256)
nms3d_kernel(int k, const float *__restrict__ corners, const float *__restrict__ score, const int *__restrict__ cls,
             const unsigned char *__restrict__ valid, float thresh, int old_type, unsigned char *__restrict__ keep) {
  extern __shared__ unsigned char smem_raw[];
  float *lo = reinterpret_cast<float *>(smem_raw);      // [k][3]
  float *hi = lo + 3 * k;                               // [k][3]
  float *vol = hi + 3 * k;                              // [k]
  float *sc = vol + k;                                  // [k]
  int *order = reinterpret_cast<int *>(sc + k);         // [k] rank -> index (candidates first, by descending score)
  int *kl = order + k;                                  // [k] class
  unsigned char *dead = reinterpret_cast<unsigned char *>(kl + k);   // [k] suppressed / not a candidate
  __shared__ int ncand;
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < k; i += blockDim.x) {
    const float *c = corners + ((size_t)b * k + i) * 24;
    float l0 = c[0], l1 = c[1], l2 = c[2], h0 = l0, h1 = l1, h2 = l2;
    for (int q = 1; q < 8; ++q) {
      l0 = fminf(l0, c[q * 3]); h0 = fmaxf(h0, c[q * 3]);
      l1 = fminf(l1, c[q * 3 + 1]); h1 = fmaxf(h1, c[q * 3 + 1]);
      l2 = fminf(l2, c[q * 3 + 2]); h2 = fmaxf(h2, c[q * 3 + 2]);
    }
    lo[3 * i] = l0; lo[3 * i + 1] = l1; lo[3 * i + 2] = l2;
    hi[3 * i] = h0; hi[3 * i + 1] = h1; hi[3 * i + 2] = h2;
    vol[i] = (h0 - l0) * (h1 - l1) * (h2 - l2);
    const float s = score[(size_t)b * k + i];
    const bool ok = valid[(size_t)b * k + i] != 0 && s == s;   // a NaN score cannot be ranked: not a candidate
    sc[i] = ok ? s : -INFINITY;
    kl[i] = cls ? cls[(size_t)b * k + i] : 0;
    dead[i] = ok ? 0 : 1;
    keep[(size_t)b * k + i] = 0;
  }
  if (tid == 0) ncand = 0;
  __syncthreads();
  // rank by counting on the pair (candidate?, score): candidates first, by descending score, ties -> higher index
  // first; then the non-candidates by index.  Candidate scores are never NaN, so this is a total order and order[]
  // a permutation of 0..k-1 whose first ncand entries are the candidates (a candidate scored -inf included).
  for (int i = tid; i < k; i += blockDim.x) {
    const float s = sc[i];
    const bool ci = !dead[i];
    int r = 0;
    for (int j = 0; j < k; ++j) {
      const float t = sc[j];
      const bool cj = !dead[j];
      r += (cj != ci) ? cj : (ci ? ((t > s) || (t == s && j > i)) : (j > i));
    }
    order[r] = i;
    if (ci) atomicAdd(&ncand, 1);
  }
  __syncthreads();
  const int nc = ncand;
  for (int a = 0; a < nc; ++a) {
    const int i = order[a];
    if (dead[i]) { __syncthreads(); continue; }      // uniform: dead[] is only written between barriers
    if (tid == 0) keep[(size_t)b * k + i] = 1;
    const float il0 = lo[3 * i], il1 = lo[3 * i + 1], il2 = lo[3 * i + 2];
    const float ih0 = hi[3 * i], ih1 = hi[3 * i + 1], ih2 = hi[3 * i + 2];
    const float vi = vol[i];
    const int ci = kl[i];
    for (int r = a + 1 + tid; r < nc; r += blockDim.x) {
      const int j = order[r];
      if (dead[j]) continue;
      const float l = fmaxf(0.f, fminf(ih0, hi[3 * j]) - fmaxf(il0, lo[3 * j]));
      const float w = fmaxf(0.f, fminf(ih1, hi[3 * j + 1]) - fmaxf(il1, lo[3 * j + 1]));
      const float h = fmaxf(0.f, fminf(ih2, hi[3 * j + 2]) - fmaxf(il2, lo[3 * j + 2]));
      const float inter = l * w * h;
      float o = old_type ? inter / vol[j] : inter / (vi + vol[j] - inter);
      if (cls && kl[j] != ci) o = 0.f;
      if (o > thresh) dead[j] = 1;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ IoU of box pairs (evaluation flavour)
__device__ __forceinline__ float edge_plain(const float *c, int i, int j) {
  const float dx = c[i * 3] - c[j * 3], dy = c[i * 3 + 1] - c[j * 3 + 1], dz = c[i * 3 + 2] - c[j * 3 + 2];
  return sqrtf(dx * dx + dy * dy + dz * dz);
}

__global__ void __launch_bounds__(128)
box3d_iou_kernel(int k1, int k2, const float *__restrict__ corners1, const float *__restrict__ corners2,
                 float *__restrict__ ious) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= k1 * k2) return;
  const int i = t / k2, j = t % k2;
  float c1[24], c2[24];
  const float *p1 = corners1 + ((size_t)b * k1 + i) * 24;
  const float *p2 = corners2 + ((size_t)b * k2 + j) * 24;
#pragma unroll
  for (int q = 0; q < 24; ++q) { c1[q] = __ldg(p1 + q); c2[q] = __ldg(p2 + q); }
  // utils/box_util.py:156-183: ground-plane rectangles from corners 3, 2, 1, 0 as (x, z); height along -y
  P2 r1[4], r2[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    r1[q] = P2{c1[(3 - q) * 3 + 0], c1[(3 - q) * 3 + 2]};
    r2[q] = P2{c2[(3 - q) * 3 + 0], c2[(3 - q) * 3 + 2]};
  }
  const float inter_area = clipped_area(r1, r2);
  const float ymax = fminf(c1[0 * 3 + 1], c2[0 * 3 + 1]);
  const float ymin = fmaxf(c1[4 * 3 + 1], c2[4 * 3 + 1]);
  const float inter_vol = inter_area * fmaxf(0.f, ymax - ymin);
  const float vol1 = edge_plain(c1, 0, 1) * edge_plain(c1, 1, 2) * edge_plain(c1, 0, 4);
  const float vol2 = edge_plain(c2, 0, 1) * edge_plain(c2, 1, 2) * edge_plain(c2, 0, 4);
  const float den = vol1 + vol2 - inter_vol;
  ious[((size_t)b * k1 + i) * k2 + j] = den > 0.f ? inter_vol / den : 0.f;
}

// ------------------------------------------------------------------ VOC matching
// One warp per (scene, class).  Detections of the scene that are in play (det_mask) are visited in descending
// score[., class] order (ties: lower index first); each looks up the ground-truth box OF THIS CLASS it overlaps
// most (first maximum, as the reference's `iou > ovmax` scan) and is a true positive iff that IoU exceeds the
// threshold and the box has not been claimed yet (utils/eval_det.py:110-146).
__global__ void __launch_bounds__(128)
eval_match_kernel(int k, int g, int ncls, const float *__restrict__ iou, const float *__restrict__ scores,
                  const unsigned char *__restrict__ det_mask, const int *__restrict__ gt_cls,
                  const unsigned char *__restrict__ gt_present, float thresh, unsigned char *__restrict__ tp) {
  extern __shared__ unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int b = blockIdx.y, c = blockIdx.x * wpb + warp;
  // per warp: order[k] ints + claimed[g] bytes
  const size_t per_warp = (size_t)k * 4 + (((size_t)g + 3) & ~(size_t)3);
  int *order = reinterpret_cast<int *>(smem_raw + warp * per_warp);
  unsigned char *claimed = reinterpret_cast<unsigned char *>(order + k);
  if (c >= ncls) return;
  const float *sc = scores + (size_t)b * k * ncls + c;          // stride ncls over detections
  const unsigned char *dm = det_mask + (size_t)b * k;
  // rank the live detections by counting (k <= a few hundred)
  // a detection of this class: in play (det_mask) and scored (a score of -inf marks "not a detection of class c")
  int nlive = 0;
  for (int i = lane; i < k; i += 32) {
    const float s = sc[(size_t)i * ncls];
    if (!dm[i] || !(s > -INFINITY)) continue;
    int r = 0;
    for (int j = 0; j < k; ++j) {
      const float t = sc[(size_t)j * ncls];
      if (!dm[j] || !(t > -INFINITY)) continue;
      r += (t > s) || (t == s && j < i);
    }
    order[r] = i;
    ++nlive;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nlive += __shfl_xor_sync(0xffffffffu, nlive, o);
  for (int j = lane; j < g; j += 32) claimed[j] = 0;
  for (int i = lane; i < k; i += 32) tp[((size_t)b * ncls + c) * k + i] = 0;
  __syncwarp();
  const int *gc = gt_cls + (size_t)b * g;
  const unsigned char *gp = gt_present + (size_t)b * g;
  for (int a = 0; a < nlive; ++a) {
    const int i = order[a];
    const float *row = iou + ((size_t)b * k + i) * g;
    float best = -INFINITY;
    int bj = -1;
    for (int j = lane; j < g; j += 32) {
      if (gp[j] && gc[j] == c) {
        const float v = row[j];
        if (v > best) { best = v; bj = j; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      // first maximum = lowest ground-truth index among equal overlaps
      if (ob > best || (ob == best && oj >= 0 && (bj < 0 || oj < bj))) { best = ob; bj = oj; }
    }
    if (lane == 0 && bj >= 0 && best > thresh && !claimed[bj]) {
      claimed[bj] = 1;
      tp[((size_t)b * ncls + c) * k + i] = 1;
    }
    __syncwarp();
  }
}

}  // namespace

extern "C" {

int coda_points_in_boxes(int b, int k, int n, int point_stride, const float *corners_camera, const float *points_depth,
                         int *counts, void *stream) {
  if (b < 0 || k < 0 || n < 0 || point_stride < 3) return CODA_EINVAL;
  if (b == 0 || k == 0) return CODA_OK;
  if (!corners_camera || !counts || (n > 0 && !points_depth) || b > 65535) return CODA_EINVAL;
  points_in_boxes_kernel<<<dim3((k + 127) / 128, b), 128, 0, (cudaStream_t)stream>>>(k, n, point_stride, corners_camera,
                                                                                  points_depth, counts);
  return launch_status();
}

int coda_nms3d(int b, int k, const float *corners, const float *score, const int *cls, const unsigned char *valid,
               float iou_thresh, int old_type, unsigned char *keep, void *stream) {
  if (b < 0 || k < 0) return CODA_EINVAL;
  if (b == 0 || k == 0) return CODA_OK;
  if (!corners || !score || !valid || !keep) return CODA_EINVAL;
  if (k > NMS_MAXK) return CODA_ETOOLARGE;
  const size_t smem = (size_t)k * (3 + 3 + 1 + 1) * 4 + (size_t)k * 8 + (size_t)k;
  static size_t configured = 0;
  if (smem > 48 * 1024 && configured < smem) {
    cudaError_t e = cudaFuncSetAttribute(nms3d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  nms3d_kernel<<<b, 256, smem, (cudaStream_t)stream>>>(k, corners, score, cls, valid, iou_thresh, old_type, keep);
  return launch_status();
}

int coda_box3d_iou(int b, int k1, int k2, const float *corners1, const float *corners2, float *ious, void *stream) {
  if (b < 0 || k1 < 0 || k2 < 0) return CODA_EINVAL;
  if (b == 0 || k1 == 0 || k2 == 0) return CODA_OK;
  if (!corners1 || !corners2 || !ious || b > 65535) return CODA_EINVAL;
  box3d_iou_kernel<<<dim3((k1 * k2 + 127) / 128, b), 128, 0, (cudaStream_t)stream>>>(k1, k2, corners1, corners2, ious);
  return launch_status();
}

int coda_eval_match(int b, int k, int g, int ncls, const float *iou, const float *scores,
                    const unsigned char *det_mask, const int *gt_cls, const unsigned char *gt_present, float iou_thresh,
                    unsigned char *tp, void *stream) {
  if (b < 0 || k < 0 || g < 0 || ncls < 0) return CODA_EINVAL;
  if (b == 0 || k == 0 || ncls == 0) return CODA_OK;
  if (!scores || !det_mask || !tp || (g > 0 && (!iou || !gt_cls || !gt_present)) || b > 65535) return CODA_EINVAL;
  const int wpb = 4;
  const size_t per_warp = (size_t)k * 4 + (((size_t)g + 3) & ~(size_t)3);
  const size_t smem = per_warp * wpb;
  if (smem > 200 * 1024) return CODA_ETOOLARGE;
  static size_t configured = 0;
  if (smem > 48 * 1024 && configured < smem) {
    cudaError_t e = cudaFuncSetAttribute(eval_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  eval_match_kernel<<<dim3((ncls + wpb - 1) / wpb, b), wpb * 32, smem, (cudaStream_t)stream>>>(
      k, g, ncls, iou, scores, det_mask, gt_cls, gt_present, iou_thresh, tp);
  return launch_status();
}

}  // extern "C"
