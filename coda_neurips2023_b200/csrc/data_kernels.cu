// Data layer on the device (sm_90a): the per-scene numpy pipeline of the reference's dataset __getitem__
// (datasets/sunrgbd_anonymous_aligned_image.py:618-795, utils/random_cuboid.py, utils/pc_util.py:24-32) and of the
// ScanNet item (datasets/scannet_anonymous_aligned_image.py:373-702) for a whole batch of raw scenes that are already
// resident in HBM:
//
//   scene_transform   flip about the YZ plane, rotation about the up axis, isotropic scale of the points
//                     (:660-705; the boxes -- a handful per scene -- follow on the host side of the module)
//   cuboid_stats      RandomCuboid (random_cuboid.py:39-95): ALL candidate crops of a scene are evaluated at once
//                     -- points inside, extent of the points inside -- one CTA per (candidate, scene)
//   cuboid_pick       the first candidate that passes the reference's tests (aspect, min_points, at least one box
//                     centre inside the extent of the kept points), or the fallback "no crop"
//   sample_points     pc_util.random_sampling: order-preserving compaction of the points inside the chosen crop, then
//                     num_points draws WITHOUT a sort: a keyed Feistel permutation of [0, M) with cycle walking
//                     (M >= num_points: without replacement; M < num_points: hashed draws with replacement), gather,
//                     and the extent of the sampled cloud (point_cloud_dims_min / max)
//   sample_points_ex  the same, plus the ScanNet item's extra gathers (positions in the cropped cloud, raw rows there)
//   flip2_rotate_scale  ScanNet: flips about YZ and XZ, rotation with a float64 matrix, float64 scale (:545-604)
//   image_augment     flip, per-channel brightness and colour shift, per-pixel jitter, clip, back to uint8 (:624-655)
//
// Randomness is the caller's: candidate tables, angles, seeds arrive as small device arrays (drawn with numpy on the
// host, like the reference draws them); the kernels are deterministic functions of them, which is what makes the CPU
// restatement (oracle/data_ref.py) bit-comparable.  Float arithmetic is written with explicit round-to-nearest
// multiplies / adds in the reference's evaluation order (no FMA contraction), so coordinates match numpy's float32.
// C-ABI in include/coda_data.h.
#include <math.h>
#include <stdint.h>

#include "../../include/coda_data.h"
#include "coda_common.cuh"

using namespace coda;

namespace {

__device__ __forceinline__ uint32_t mix32d(uint32_t h) {
  h ^= h >> 16; h *= 0x7FEB352Du; h ^= h >> 15; h *= 0x846CA68Bu; h ^= h >> 16;
  return h;
}

// coordinate-type helpers: the float32 instantiations keep the exact operations they were written with (fminf /
// fmaxf, __double2float_rn), the float64 ones (SUN RGB-D's float64 scene files) the same operations on doubles
__device__ __forceinline__ float vmin(float a, float b) { return fminf(a, b); }
__device__ __forceinline__ float vmax(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double vmin(double a, double b) { return fmin(a, b); }
__device__ __forceinline__ double vmax(double a, double b) { return fmax(a, b); }
template <typename T> __device__ __forceinline__ T from_double(double v);
template <> __device__ __forceinline__ float from_double<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double from_double<double>(double v) { return v; }

// ------------------------------------------------------------------ flip / rotate / scale
// xyz' = ((flip_x * x, y, z) @ rot^T) * scale, evaluated as numpy does on float32 arrays: products and sums rounded
// separately, left to right (datasets/...:663-700: point_cloud[:, 0] *= -1; np.dot(pc, rot^T); pc *= scale)
__global__ void __launch_bounds__(256)
scene_transform_kernel(int nmax, int stride, const int *__restrict__ npts, const float *__restrict__ flip,
                       const float *__restrict__ rot, const float *__restrict__ scale, float *__restrict__ pts) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npts[b] || i >= nmax) return;
  float *p = pts + ((size_t)b * nmax + i) * stride;
  const float *R = rot + b * 9;
  const float x = __fmul_rn(p[0], flip[b]), y = p[1], z = p[2];
  const float s = scale[b];
  // (x, y, z) @ rot^T  ->  component j = x R[j][0] + y R[j][1] + z R[j][2]
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float v = __fadd_rn(__fadd_rn(__fmul_rn(x, R[j * 3]), __fmul_rn(y, R[j * 3 + 1])), __fmul_rn(z, R[j * 3 + 2]));
    p[j] = __fmul_rn(v, s);
  }
}

// ------------------------------------------------------------------ RandomCuboid
// stats[b][c] = {count, min x, min y, min z, max x, max y, max z} of the points inside candidate c
// (random_cuboid.py:47-66: centre = a point of the cloud, half extent = range_xyz * crop_range / 2, inclusive bounds)
template <typename T>
__global__ void __launch_bounds__(256)
cuboid_stats_kernel(int nmax, int stride, int ncand, const int *__restrict__ npts, const T *__restrict__ pts,
                    const T *__restrict__ range_xyz, const double *__restrict__ crop_range,
                    const float *__restrict__ center_u, T *__restrict__ stats) {
  const int b = blockIdx.y, c = blockIdx.x, n = min(npts[b], nmax);
  const T *P = pts + (size_t)b * nmax * stride;
  const double *cr = crop_range + ((size_t)b * ncand + c) * 3;
  int ci = (int)(center_u[(size_t)b * ncand + c] * (float)n);
  ci = ci < 0 ? 0 : (ci >= n ? n - 1 : ci);
  // the reference mixes float32 points with float64 random numbers: the bounds are doubles (random_cuboid.py:55-58)
  double lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double half = (double)range_xyz[b * 3 + a] * cr[a] / 2.0;
    const double ctr = n > 0 ? (double)P[(size_t)ci * stride + a] : 0.0;
    lo[a] = ctr - half;
    hi[a] = ctr + half;
  }
  int cnt = 0;
  T mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const T x = P[(size_t)i * stride], y = P[(size_t)i * stride + 1], z = P[(size_t)i * stride + 2];
    if ((double)x <= hi[0] && (double)y <= hi[1] && (double)z <= hi[2] && (double)x >= lo[0] && (double)y >= lo[1] &&
        (double)z >= lo[2]) {
      ++cnt;
      mn[0] = vmin(mn[0], x); mn[1] = vmin(mn[1], y); mn[2] = vmin(mn[2], z);
      mx[0] = vmax(mx[0], x); mx[1] = vmax(mx[1], y); mx[2] = vmax(mx[2], z);
    }
  }
  __shared__ int s_cnt[8];
  __shared__ T s_mn[8][3], s_mx[8][3];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      mn[a] = vmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = vmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    s_cnt[w] = cnt;
    for (int a = 0; a < 3; ++a) { s_mn[w][a] = mn[a]; s_mx[w][a] = mx[a]; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < (int)(blockDim.x >> 5); ++q) {
      cnt += s_cnt[q];
      for (int a = 0; a < 3; ++a) { mn[a] = vmin(mn[a], s_mn[q][a]); mx[a] = vmax(mx[a], s_mx[q][a]); }
    }
    T *o = stats + ((size_t)b * ncand + c) * 8;
    o[0] = (T)cnt;
    for (int a = 0; a < 3; ++a) { o[1 + a] = mn[a]; o[4 + a] = mx[a]; }
    o[7] = 0;
  }
}

// chosen[b] = index of the first candidate that passes every test of random_cuboid.py:42-86, or -1 (fallback:
// the scene is kept whole); box_keep (b, gmax) = boxes whose centre lies within the extent of the kept points;
// crop (b, 6) = the chosen cuboid's inclusive bounds (lo xyz, hi xyz)
template <typename T>
__global__ void __launch_bounds__(32)
cuboid_pick_kernel(int nmax, int stride, int ncand, int gmax, int min_points, float aspect_min,
                   const int *__restrict__ npts, const T *__restrict__ pts, const T *__restrict__ range_xyz,
                   const double *__restrict__ crop_range, const float *__restrict__ center_u,
                   const T *__restrict__ stats, const T *__restrict__ boxes, int box_stride,
                   const int *__restrict__ nbox, int *__restrict__ chosen, double *__restrict__ crop,
                   unsigned char *__restrict__ box_keep) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int n = min(npts[b], nmax), ng = min(nbox[b], gmax);
  const T *B = boxes + (size_t)b * gmax * box_stride;
  // "target_boxes.sum() > 0": ground truth present at all (random_cuboid.py:74), summed in the boxes' type
  T bsum = 0;
  for (int i = lane; i < ng * box_stride; i += 32) bsum += B[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bsum += __shfl_xor_sync(0xffffffffu, bsum, o);
  const bool has_boxes = bsum > (T)0;
  int pick = -1;
  for (int c0 = 0; c0 < ncand && pick < 0; c0 += 32) {
    const int c = c0 + lane;
    bool ok = false;
    if (c < ncand && n > 0) {
      const double *cr = crop_range + ((size_t)b * ncand + c) * 3;
      const double xy = fmin(cr[0], cr[1]) / fmax(cr[0], cr[1]);
      const double xz = fmin(cr[0], cr[2]) / fmax(cr[0], cr[2]);
      const double yz = fmin(cr[1], cr[2]) / fmax(cr[1], cr[2]);
      const T *st = stats + ((size_t)b * ncand + c) * 8;
      ok = (xy >= (double)aspect_min || xz >= (double)aspect_min || yz >= (double)aspect_min) && (int)st[0] >= min_points;
      if (ok && has_boxes) {
        bool any = false;
        for (int q = 0; q < ng; ++q) {
          const T *bx = B + (size_t)q * box_stride;
          any = any || (bx[0] >= st[1] && bx[1] >= st[2] && bx[2] >= st[3] && bx[0] <= st[4] && bx[1] <= st[5] && bx[2] <= st[6]);
        }
        ok = any;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (m) pick = c0 + __ffs(m) - 1;
  }
  if (lane == 0) chosen[b] = pick;
  double lo[3] = {-INFINITY, -INFINITY, -INFINITY}, hi[3] = {INFINITY, INFINITY, INFINITY};
  const T *st = pick >= 0 ? stats + ((size_t)b * ncand + pick) * 8 : nullptr;
  if (pick >= 0) {
    const T *P = pts + (size_t)b * nmax * stride;
    const double *cr = crop_range + ((size_t)b * ncand + pick) * 3;
    int ci = (int)(center_u[(size_t)b * ncand + pick] * (float)n);
    ci = ci < 0 ? 0 : (ci >= n ? n - 1 : ci);
    for (int a = 0; a < 3; ++a) {
      const double half = (double)range_xyz[b * 3 + a] * cr[a] / 2.0;
      lo[a] = (double)P[(size_t)ci * stride + a] - half;
      hi[a] = (double)P[(size_t)ci * stride + a] + half;
    }
  }
  if (lane < 3) { crop[b * 6 + lane] = lo[lane]; crop[b * 6 + 3 + lane] = hi[lane]; }
  for (int q = lane; q < gmax; q += 32) {
    bool keep = q < ng;
    if (keep && pick >= 0 && has_boxes) {
      const T *bx = B + (size_t)q * box_stride;
      keep = bx[0] >= st[1] && bx[1] >= st[2] && bx[2] >= st[3] && bx[0] <= st[4] && bx[1] <= st[5] && bx[2] <= st[6];
    }
    box_keep[(size_t)b * gmax + q] = keep ? 1 : 0;
  }
}

// ------------------------------------------------------------------ compaction + sampling
// order-preserving list of the points inside crop[b]: one CTA per scene, block scan per 1024-point chunk
template <typename T>
__global__ void __launch_bounds__(1024)
compact_kernel(int nmax, int stride, const int *__restrict__ npts, const T *__restrict__ pts,
               const double *__restrict__ crop, int *__restrict__ list, int *__restrict__ count) {
  __shared__ int warp_sum[32];
  __shared__ int base;
  const int b = blockIdx.x, n = min(npts[b], nmax), lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const T *P = pts + (size_t)b * nmax * stride;
  const double *cb = crop + b * 6;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    bool in = false;
    if (i < n) {
      const T x = P[(size_t)i * stride], y = P[(size_t)i * stride + 1], z = P[(size_t)i * stride + 2];
      in = (double)x <= cb[3] && (double)y <= cb[4] && (double)z <= cb[5] && (double)x >= cb[0] && (double)y >= cb[1] &&
           (double)z >= cb[2];
    }
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (lane == 0) warp_sum[w] = __popc(m);
    __syncthreads();
    int off = base;
    for (int q = 0; q < w; ++q) off += warp_sum[q];
    if (in) list[(size_t)b * nmax + off + __popc(m & ((1u << lane) - 1))] = i;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int q = 0; q < 32; ++q) t += warp_sum[q];
      base += t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[b] = base;
}

// keyed bijection of [0, 2^bits): four Feistel rounds on the two halves of the index
__device__ __forceinline__ uint32_t feistel(uint32_t x, int half_bits, uint32_t key) {
  const uint32_t mask = (1u << half_bits) - 1u;
  uint32_t l = x >> half_bits, r = x & mask;
#pragma unroll
  for (int round = 0; round < 4; ++round) {
    const uint32_t f = mix32d(r * 0x9E3779B1u + key + (uint32_t)round * 0x85EBCA6Bu) & mask;
    const uint32_t nl = r;
    r = l ^ f;
    l = nl;
  }
  return (l << half_bits) | r;
}

// out[b][i] = points[list[perm_b(i)]]  (all `stride` columns), i < nsample.  M >= nsample: perm = Feistel bijection
// on the next power of four >= M, cycle-walked back into [0, M) -- distinct indices, no sort.  M < nsample: hashed
// draws (with replacement, like np.random.choice(..., replace=True)).  choice (b, nsample) = index into the raw scene.
// kEx (the ScanNet item, datasets/scannet_anonymous_aligned_image.py:507-532) also writes list_pos = perm_b(i), the
// position in the cropped cloud, and rgb_out[b][i] = the first rgb_stride columns of the RAW scene's row list_pos --
// the reference indexes the uncropped scene with the cropped cloud's choices.
template <typename T, bool kEx>
__global__ void __launch_bounds__(256)
sample_kernel(int nmax, int stride, int nsample, const T *__restrict__ pts, const int *__restrict__ list,
              const int *__restrict__ count, const uint32_t *__restrict__ seed, T *__restrict__ out,
              int *__restrict__ choice, int rgb_stride, int *__restrict__ list_pos, T *__restrict__ rgb_out) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nsample) return;
  const int m = count[b];
  int src = 0;
  uint32_t j = 0;
  if (m > 0) {
    const uint32_t key = mix32d(seed[b] ^ 0xA511E9B3u);
    if (m >= nsample) {
      int half_bits = 1;
      while ((1u << (2 * half_bits)) < (uint32_t)m) ++half_bits;
      j = (uint32_t)i;
      do { j = feistel(j, half_bits, key); } while (j >= (uint32_t)m);      // cycle walking
    } else {
      j = mix32d((uint32_t)i * 0x9E3779B1u + key) % (uint32_t)m;
    }
    src = list[(size_t)b * nmax + j];
  }
  const T *p = pts + ((size_t)b * nmax + src) * stride;
  T *o = out + ((size_t)b * nsample + i) * stride;
  for (int c = 0; c < stride; ++c) o[c] = m > 0 ? p[c] : (T)0;
  choice[(size_t)b * nsample + i] = m > 0 ? src : -1;
  if (kEx) {
    const T *q = pts + ((size_t)b * nmax + j) * stride;
    T *r = rgb_out + ((size_t)b * nsample + i) * rgb_stride;
    for (int c = 0; c < rgb_stride; ++c) r[c] = m > 0 ? q[c] : (T)0;
    list_pos[(size_t)b * nsample + i] = m > 0 ? (int)j : -1;
  }
}

// ------------------------------------------------------------------ ScanNet flips / rotation / scale
// datasets/scannet_anonymous_aligned_image.py:545-604 on float32 rows: x <- -x (YZ flip), y <- -y (XZ flip), exact;
// then np.dot(pc[:, 0:3], rot^T) with a float64 rot -- numpy promotes to float64 and BLAS accumulates the three
// products with fused multiply-adds, the result is stored back as float32 -- and finally `pc[:, 0:3] *= scale`
// with a float64 scale: float64 product, stored as float32.  On float64 rows (SUN RGB-D's scene files,
// datasets/sunrgbd_anonymous_aligned_image.py:664-709) the same statements run in float64 end to end: the same fused
// chain, no rounding between the rotation and the scale.  The flips are exact in both types.
template <typename T>
__global__ void __launch_bounds__(256)
flip2_rotate_scale_kernel(int nmax, int stride, const int *__restrict__ npts, const float *__restrict__ flip_yz,
                          const float *__restrict__ flip_xz, const double *__restrict__ rot,
                          const double *__restrict__ scale, T *__restrict__ pts) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nmax || (npts && i >= npts[b])) return;
  T *p = pts + ((size_t)b * nmax + i) * stride;
  const double *R = rot + b * 9;
  const double x = (double)(p[0] * (T)flip_yz[b]), y = (double)(p[1] * (T)flip_xz[b]), z = (double)p[2];
  const double s = scale[b];
  T v[3];
#pragma unroll
  for (int j = 0; j < 3; ++j)
    v[j] = from_double<T>(__fma_rn(z, R[j * 3 + 2], __fma_rn(y, R[j * 3 + 1], __dmul_rn(x, R[j * 3]))));
#pragma unroll
  for (int j = 0; j < 3; ++j) p[j] = from_double<T>(__dmul_rn((double)v[j], s));
}

// per-scene extent of the first three columns: dims (b, 6) = min xyz | max xyz
template <typename T>
__global__ void __launch_bounds__(256)
extent_kernel(int nmax, int stride, const int *__restrict__ npts, const T *__restrict__ pts, T *__restrict__ dims) {
  const int b = blockIdx.x;
  const int n = npts ? min(npts[b], nmax) : nmax;
  const T *P = pts + (size_t)b * nmax * stride;
  T mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const T v = P[(size_t)i * stride + a];
      mn[a] = vmin(mn[a], v);
      mx[a] = vmax(mx[a], v);
    }
  }
  __shared__ T s_mn[8][3], s_mx[8][3];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      mn[a] = vmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = vmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int a = 0; a < 3; ++a) { s_mn[w][a] = mn[a]; s_mx[w][a] = mx[a]; }
  __syncthreads();
  if (threadIdx.x < 3) {
    T lo = s_mn[0][threadIdx.x], hi = s_mx[0][threadIdx.x];
    for (int q = 1; q < (int)(blockDim.x >> 5); ++q) { lo = vmin(lo, s_mn[q][threadIdx.x]); hi = vmax(hi, s_mx[q][threadIdx.x]); }
    dims[b * 6 + threadIdx.x] = lo;
    dims[b * 6 + 3 + threadIdx.x] = hi;
  }
}

// ------------------------------------------------------------------ image augmentation
// datasets/...:624-655 on uint8 HWC images: /255, horizontal flip, per-channel gain and shift, per-pixel jitter,
// clip to [0, 1], * 255, truncation to uint8.  gain / shift (b, 3); jitter = 0.05 u - 0.025 with u from a counter hash.
__global__ void __launch_bounds__(256)
image_augment_kernel(int h, int w, const unsigned char *__restrict__ in, const unsigned char *__restrict__ flip,
                     const float *__restrict__ gain, const float *__restrict__ shift, const uint32_t *__restrict__ seed,
                     unsigned char *__restrict__ out) {
  const int b = blockIdx.y;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)h * w) return;
  const int y = (int)(t / w), x = (int)(t % w);
  const int sx = flip[b] ? w - 1 - x : x;
  const unsigned char *p = in + (((size_t)b * h + y) * w + sx) * 3;
  unsigned char *o = out + (((size_t)b * h + y) * w + x) * 3;
  const uint32_t r = mix32d(seed[b] + (uint32_t)t * 0x9E3779B1u);
  const float jit = __fsub_rn(__fmul_rn(0.05f, (float)(r >> 8) * (1.0f / 16777216.0f)), 0.025f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = __fdiv_rn((float)p[c], 255.0f);
    v = __fmul_rn(v, gain[b * 3 + c]);
    v = __fadd_rn(v, shift[b * 3 + c]);
    v = __fadd_rn(v, jit);
    v = fminf(fmaxf(v, 0.f), 1.f);
    o[c] = (unsigned char)(__fmul_rn(v, 255.0f));
  }
}

// ------------------------------------------------------------------ host launchers shared by the fp32 / fp64 entry points
template <typename T>
int random_cuboid(int b, int nmax, int stride, int ncand, int gmax, int box_stride, int min_points, float aspect_min,
                  const int *npts, const T *points, const T *range_xyz, const double *crop_range, const float *center_u,
                  const T *boxes, const int *nbox, T *stats_scratch, int *chosen, double *crop,
                  unsigned char *box_keep, void *stream) {
  if (b < 0 || nmax <= 0 || stride < 3 || ncand <= 0 || gmax < 0 || box_stride < 3) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!npts || !points || !range_xyz || !crop_range || !center_u || !nbox || !stats_scratch || !chosen || !crop ||
      (gmax > 0 && (!boxes || !box_keep)) || b > 65535)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  cuboid_stats_kernel<T><<<dim3(ncand, b), 256, 0, s>>>(nmax, stride, ncand, npts, points, range_xyz, crop_range,
                                                        center_u, stats_scratch);
  cuboid_pick_kernel<T><<<b, 32, 0, s>>>(nmax, stride, ncand, gmax, min_points, aspect_min, npts, points, range_xyz,
                                         crop_range, center_u, stats_scratch, boxes, box_stride, nbox, chosen, crop,
                                         box_keep);
  return launch_status();
}

template <typename T>
int sample_points(int b, int nmax, int stride, int nsample, const int *npts, const T *points, const double *crop,
                  const unsigned int *seed, int *list_scratch, int *count, T *out, int *choice, T *dims,
                  void *stream) {
  if (b < 0 || nmax <= 0 || stride < 3 || nsample <= 0) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!npts || !points || !crop || !seed || !list_scratch || !count || !out || !choice || !dims || b > 65535)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  compact_kernel<T><<<b, 1024, 0, s>>>(nmax, stride, npts, points, crop, list_scratch, count);
  sample_kernel<T, false><<<dim3((nsample + 255) / 256, b), 256, 0, s>>>(nmax, stride, nsample, points, list_scratch,
                                                                         count, seed, out, choice, 0, nullptr, nullptr);
  extent_kernel<T><<<b, 256, 0, s>>>(nsample, stride, nullptr, out, dims);
  return launch_status();
}

template <typename T>
int flip2_rotate_scale(int b, int nmax, int stride, const int *npts, const float *flip_yz, const float *flip_xz,
                       const double *rot, const double *scale, T *points, void *stream) {
  if (b < 0 || nmax < 0 || stride < 3) return CODA_EINVAL;
  if (b == 0 || nmax == 0) return CODA_OK;
  if (!flip_yz || !flip_xz || !rot || !scale || !points || b > 65535) return CODA_EINVAL;
  flip2_rotate_scale_kernel<T><<<dim3((nmax + 255) / 256, b), 256, 0, (cudaStream_t)stream>>>(
      nmax, stride, npts, flip_yz, flip_xz, rot, scale, points);
  return launch_status();
}

template <typename T>
int points_extent(int b, int nmax, int stride, const int *npts, const T *points, T *dims, void *stream) {
  if (b < 0 || nmax <= 0 || stride < 3) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!points || !dims) return CODA_EINVAL;
  extent_kernel<T><<<b, 256, 0, (cudaStream_t)stream>>>(nmax, stride, npts, points, dims);
  return launch_status();
}

}  // namespace

extern "C" {

int coda_scene_transform(int b, int nmax, int stride, const int *npts, const float *flip, const float *rot,
                         const float *scale, float *points, void *stream) {
  if (b < 0 || nmax < 0 || stride < 3) return CODA_EINVAL;
  if (b == 0 || nmax == 0) return CODA_OK;
  if (!npts || !flip || !rot || !scale || !points || b > 65535) return CODA_EINVAL;
  scene_transform_kernel<<<dim3((nmax + 255) / 256, b), 256, 0, (cudaStream_t)stream>>>(nmax, stride, npts, flip, rot,
                                                                                      scale, points);
  return launch_status();
}

int coda_random_cuboid(int b, int nmax, int stride, int ncand, int gmax, int box_stride, int min_points,
                       float aspect_min, const int *npts, const float *points, const float *range_xyz,
                       const double *crop_range, const float *center_u, const float *boxes, const int *nbox,
                       float *stats_scratch, int *chosen, double *crop, unsigned char *box_keep, void *stream) {
  return random_cuboid<float>(b, nmax, stride, ncand, gmax, box_stride, min_points, aspect_min, npts, points, range_xyz,
                              crop_range, center_u, boxes, nbox, stats_scratch, chosen, crop, box_keep, stream);
}

int coda_random_cuboid_f64(int b, int nmax, int stride, int ncand, int gmax, int box_stride, int min_points,
                           float aspect_min, const int *npts, const double *points, const double *range_xyz,
                           const double *crop_range, const float *center_u, const double *boxes, const int *nbox,
                           double *stats_scratch, int *chosen, double *crop, unsigned char *box_keep, void *stream) {
  return random_cuboid<double>(b, nmax, stride, ncand, gmax, box_stride, min_points, aspect_min, npts, points,
                               range_xyz, crop_range, center_u, boxes, nbox, stats_scratch, chosen, crop, box_keep,
                               stream);
}

int coda_sample_points(int b, int nmax, int stride, int nsample, const int *npts, const float *points,
                       const double *crop, const unsigned int *seed, int *list_scratch, int *count, float *out,
                       int *choice, float *dims, void *stream) {
  return sample_points<float>(b, nmax, stride, nsample, npts, points, crop, seed, list_scratch, count, out, choice,
                              dims, stream);
}

int coda_sample_points_f64(int b, int nmax, int stride, int nsample, const int *npts, const double *points,
                           const double *crop, const unsigned int *seed, int *list_scratch, int *count, double *out,
                           int *choice, double *dims, void *stream) {
  return sample_points<double>(b, nmax, stride, nsample, npts, points, crop, seed, list_scratch, count, out, choice,
                               dims, stream);
}

int coda_sample_points_ex(int b, int nmax, int stride, int nsample, int rgb_stride, const int *npts,
                          const float *points, const double *crop, const unsigned int *seed, int *list_scratch,
                          int *count, float *out, int *choice, int *list_pos, float *rgb_out, float *dims,
                          void *stream) {
  if (b < 0 || nmax <= 0 || stride < 3 || nsample <= 0 || rgb_stride < 0 || rgb_stride > stride) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!npts || !points || !crop || !seed || !list_scratch || !count || !out || !choice || !list_pos || !dims ||
      (rgb_stride > 0 && !rgb_out) || b > 65535)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  compact_kernel<float><<<b, 1024, 0, s>>>(nmax, stride, npts, points, crop, list_scratch, count);
  sample_kernel<float, true><<<dim3((nsample + 255) / 256, b), 256, 0, s>>>(nmax, stride, nsample, points,
                                                                            list_scratch, count, seed, out, choice,
                                                                            rgb_stride, list_pos, rgb_out);
  extent_kernel<float><<<b, 256, 0, s>>>(nsample, stride, nullptr, out, dims);
  return launch_status();
}

int coda_points_flip2_rotate_scale(int b, int nmax, int stride, const int *npts, const float *flip_yz,
                                   const float *flip_xz, const double *rot, const double *scale, float *points,
                                   void *stream) {
  return flip2_rotate_scale<float>(b, nmax, stride, npts, flip_yz, flip_xz, rot, scale, points, stream);
}

int coda_points_flip2_rotate_scale_f64(int b, int nmax, int stride, const int *npts, const float *flip_yz,
                                       const float *flip_xz, const double *rot, const double *scale, double *points,
                                       void *stream) {
  return flip2_rotate_scale<double>(b, nmax, stride, npts, flip_yz, flip_xz, rot, scale, points, stream);
}

int coda_points_extent(int b, int nmax, int stride, const int *npts, const float *points, float *dims, void *stream) {
  return points_extent<float>(b, nmax, stride, npts, points, dims, stream);
}

int coda_points_extent_f64(int b, int nmax, int stride, const int *npts, const double *points, double *dims,
                           void *stream) {
  return points_extent<double>(b, nmax, stride, npts, points, dims, stream);
}

int coda_image_augment(int b, int h, int w, const unsigned char *in, const unsigned char *flip, const float *gain,
                       const float *shift, const unsigned int *seed, unsigned char *out, void *stream) {
  if (b < 0 || h < 0 || w < 0) return CODA_EINVAL;
  if (b == 0 || h == 0 || w == 0) return CODA_OK;
  if (!in || !flip || !gain || !shift || !seed || !out || in == out || b > 65535) return CODA_EINVAL;
  const long long px = (long long)h * w;
  image_augment_kernel<<<dim3((unsigned)((px + 255) / 256), b), 256, 0, (cudaStream_t)stream>>>(h, w, in, flip, gain,
                                                                                             shift, seed, out);
  return launch_status();
}

}  // extern "C"
