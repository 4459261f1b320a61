// Warp-primitive kernels of the 3DETR encoder/decoder and of the matcher for
// H100 (sm_90a): LayerNorm fwd/bwd, row softmax, fused Fourier positional
// encoding, generalised 3-D IoU with rotated-rectangle clipping, and a
// warp-per-scene Hungarian solver.  C-ABI in include/coda_detr.h.
#include <cuda_fp16.h>
#include <math.h>

#include "../../include/coda_detr.h"
#include "coda_common.cuh"
#include "box_geometry.cuh"

using namespace coda;

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// =====================================================================
//  LayerNorm: one warp per row, the row lives in registers (NV float4 / lane)
// =====================================================================
constexpr int LN_WARPS = 8;

// Where row r of a (rows, c) operand lives: r * c when inner == 0, else (r / inner) * so + (r % inner) * si floats --
// a (q, b) -> (b, q) row permutation or a slice of a larger buffer costs no copy.
struct RowMap {
  int inner;
  long long so, si;
};
__device__ __forceinline__ long long map_row(const RowMap &m, long long r, int c) {
  return m.inner ? (r / m.inner) * m.so + (r % m.inner) * m.si : r * c;
}

// y = LayerNorm(x) (optional, row-mapped); ypos = y + pos (optional): the `norm(x) + query_pos` operand of the
// decoder's attention comes out of the same pass.
template <int NV>  // c == NV * 128
__global__ void __launch_bounds__(LN_WARPS * 32)
layer_norm_fwd_kernel(long long rows, float eps, const float *__restrict__ x,
                      const float *__restrict__ gamma, const float *__restrict__ beta,
                      float *__restrict__ y, const RowMap ymap, const float *__restrict__ pos,
                      float *__restrict__ ypos, float *__restrict__ mean_out,
                      float *__restrict__ rstd_out) {
  constexpr int C = NV * 128;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4 *xr = reinterpret_cast<const float4 *>(x + row * C);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] = __ldg(xr + lane + i * 32);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float var = warp_sum(q) * (1.0f / C);
  const float rstd = 1.0f / sqrtf(var + eps);
  float4 *yr = y ? reinterpret_cast<float4 *>(y + map_row(ymap, row, C)) : nullptr;
  const float4 *pr = pos ? reinterpret_cast<const float4 *>(pos + row * C) : nullptr;
  float4 *ypr = pos ? reinterpret_cast<float4 *>(ypos + row * C) : nullptr;
  const float4 *g4 = reinterpret_cast<const float4 *>(gamma);
  const float4 *b4 = reinterpret_cast<const float4 *>(beta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = __ldg(g4 + lane + i * 32), b = __ldg(b4 + lane + i * 32);
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + b.x;
    o.y = (v[i].y - mean) * rstd * g.y + b.y;
    o.z = (v[i].z - mean) * rstd * g.z + b.z;
    o.w = (v[i].w - mean) * rstd * g.w + b.w;
    if (yr) yr[lane + i * 32] = o;
    if (pr) {
      const float4 pv = __ldg(pr + lane + i * 32);
      ypr[lane + i * 32] = make_float4(o.x + pv.x, o.y + pv.y, o.z + pv.z, o.w + pv.w);
    }
  }
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
}

// fp16 activations (CLIP towers): same statistics in fp32, half in / half out
template <int NV>  // c == NV * 128
__global__ void __launch_bounds__(LN_WARPS * 32)
layer_norm_fwd_half_kernel(long long rows, float eps, const __half *__restrict__ x,
                           const float *__restrict__ gamma, const float *__restrict__ beta,
                           __half *__restrict__ y) {
  constexpr int C = NV * 128;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * LN_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint2 *xr = reinterpret_cast<const uint2 *>(x + row * C);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const uint2 raw = __ldg(xr + lane + i * 32);
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
    v[i] = make_float4(lo.x, lo.y, hi.x, hi.y);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / C) + eps);
  uint2 *yr = reinterpret_cast<uint2 *>(y + row * C);
  const float4 *g4 = reinterpret_cast<const float4 *>(gamma);
  const float4 *b4 = reinterpret_cast<const float4 *>(beta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 g = __ldg(g4 + lane + i * 32), b = __ldg(b4 + lane + i * 32);
    const __half2 lo = __floats2half2_rn((v[i].x - mean) * rstd * g.x + b.x, (v[i].y - mean) * rstd * g.y + b.y);
    const __half2 hi = __floats2half2_rn((v[i].z - mean) * rstd * g.z + b.z, (v[i].w - mean) * rstd * g.w + b.w);
    uint2 o;
    o.x = *reinterpret_cast<const unsigned *>(&lo);
    o.y = *reinterpret_cast<const unsigned *>(&hi);
    yr[lane + i * 32] = o;
  }
}

constexpr int LN_BWD_ROWS_PER_BLOCK = 64;  // each warp walks 8 rows

// d = dy (row-mapped) + dy2 (optional: the gradient that arrived through the `+ pos` output);
// dx = LayerNormBackward(d) + add (optional: the gradient of the residual branch that by-passes the norm)
template <int NV>
__global__ void __launch_bounds__(LN_WARPS * 32)
layer_norm_bwd_kernel(long long rows, const float *__restrict__ dy, const RowMap dmap,
                      const float *__restrict__ dy2, const float *__restrict__ add,
                      const float *__restrict__ x,
                      const float *__restrict__ gamma, const float *__restrict__ mean,
                      const float *__restrict__ rstd, float *__restrict__ dx,
                      float *__restrict__ partial) {
  constexpr int C = NV * 128;
  __shared__ float4 red[LN_WARPS][NV * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float4 *g4 = reinterpret_cast<const float4 *>(gamma);
  float4 g[NV], dg[NV], db[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    g[i] = __ldg(g4 + lane + i * 32);
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const long long row0 = (long long)blockIdx.x * LN_BWD_ROWS_PER_BLOCK;
  for (int r = warp; r < LN_BWD_ROWS_PER_BLOCK; r += LN_WARPS) {
    const long long row = row0 + r;
    if (row >= rows) break;
    const float m = __ldg(mean + row), rs = __ldg(rstd + row);
    const float4 *xr = reinterpret_cast<const float4 *>(x + row * C);
    const float4 *dr = reinterpret_cast<const float4 *>(dy + map_row(dmap, row, C));
    const float4 *d2r = dy2 ? reinterpret_cast<const float4 *>(dy2 + row * C) : nullptr;
    const float4 *ar = add ? reinterpret_cast<const float4 *>(add + row * C) : nullptr;
    float4 xh[NV], d[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 xv = __ldg(xr + lane + i * 32);
      d[i] = __ldg(dr + lane + i * 32);
      if (d2r) {
        const float4 t = __ldg(d2r + lane + i * 32);
        d[i].x += t.x; d[i].y += t.y; d[i].z += t.z; d[i].w += t.w;
      }
      xh[i] = make_float4((xv.x - m) * rs, (xv.y - m) * rs, (xv.z - m) * rs, (xv.w - m) * rs);
      dg[i].x += d[i].x * xh[i].x; dg[i].y += d[i].y * xh[i].y;
      dg[i].z += d[i].z * xh[i].z; dg[i].w += d[i].w * xh[i].w;
      db[i].x += d[i].x; db[i].y += d[i].y; db[i].z += d[i].z; db[i].w += d[i].w;
      d[i].x *= g[i].x; d[i].y *= g[i].y; d[i].z *= g[i].z; d[i].w *= g[i].w;  // dxhat
      s1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
      s2 += (d[i].x * xh[i].x + d[i].y * xh[i].y) + (d[i].z * xh[i].z + d[i].w * xh[i].w);
    }
    const float c1 = warp_sum(s1) * (1.0f / C), c2 = warp_sum(s2) * (1.0f / C);
    float4 *dxr = reinterpret_cast<float4 *>(dx + row * C);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float4 o;
      o.x = rs * (d[i].x - c1 - xh[i].x * c2);
      o.y = rs * (d[i].y - c1 - xh[i].y * c2);
      o.z = rs * (d[i].z - c1 - xh[i].z * c2);
      o.w = rs * (d[i].w - c1 - xh[i].w * c2);
      if (ar) {
        const float4 t = __ldg(ar + lane + i * 32);
        o.x += t.x; o.y += t.y; o.z += t.z; o.w += t.w;
      }
      dxr[lane + i * 32] = o;
    }
  }
  // block reduction of the per-warp column sums, one partial row per block:
  // partial[blk][0][c] = dgamma, partial[blk][1][c] = dbeta
  float4 *pg = reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * 2 * C);
  float4 *pb = pg + NV * 32;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp][lane + i * 32] = pass == 0 ? dg[i] : db[i];
    __syncthreads();
    for (int col = threadIdx.x; col < NV * 32; col += LN_WARPS * 32) {
      float4 a = red[0][col];
#pragma unroll
      for (int w = 1; w < LN_WARPS; ++w) {
        const float4 t = red[w][col];
        a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
      }
      (pass == 0 ? pg : pb)[col] = a;
    }
  }
}

__global__ void layer_norm_bwd_finalize(int nblocks, int c, const float *__restrict__ partial,
                                        float *__restrict__ dgamma, float *__restrict__ dbeta) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= 2 * c) return;
  float a = 0.f;
  for (int blk = 0; blk < nblocks; ++blk) a += partial[(size_t)blk * 2 * c + col];
  if (col < c) dgamma[col] = a; else dbeta[col - c] = a;
}

// =====================================================================
//  Row softmax (any width), one warp per row
// =====================================================================
__global__ void __launch_bounds__(256)
softmax_rows_kernel(long long rows, int c, int log_softmax, const float *__restrict__ x,
                    float *__restrict__ y) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float *xr = x + row * c;
  float *yr = y + row * c;
  float m = -INFINITY;
  for (int i = lane; i < c; i += 32) m = fmaxf(m, __ldg(xr + i));
  m = warp_max(m);
  float s = 0.f;
  for (int i = lane; i < c; i += 32) s += expf(__ldg(xr + i) - m);
  s = warp_sum(s);
  if (log_softmax) {
    const float ls = logf(s);
    for (int i = lane; i < c; i += 32) yr[i] = (__ldg(xr + i) - m) - ls;
  } else {
    const float inv = 1.0f / s;
    for (int i = lane; i < c; i += 32) yr[i] = expf(__ldg(xr + i) - m) * inv;
  }
}

// =====================================================================
//  Fourier positional encoding
// =====================================================================
// grid (ceil(n / 128), ceil(d_out / FOURIER_CH), b); thread = one point, loops
// over a slab of channels; stores are coalesced along n for every channel.
constexpr int FOURIER_CH = 32;

__global__ void __launch_bounds__(128)
fourier_kernel(int n, int d_out, int ldb, int normalize, const float *__restrict__ xyz,
               const float *__restrict__ rmin, const float *__restrict__ rmax,
               const float *__restrict__ gauss_b, float *__restrict__ out) {
  __shared__ float sB[3][FOURIER_CH];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * FOURIER_CH;
  const int nc = min(FOURIER_CH, d_out - c0);
  if (threadIdx.x < 3 * FOURIER_CH) {
    const int d = threadIdx.x / FOURIER_CH, c = threadIdx.x % FOURIER_CH;
    sB[d][c] = c < nc ? __ldg(gauss_b + (size_t)d * ldb + c0 + c) : 0.f;
  }
  __syncthreads();
  const int p = blockIdx.x * 128 + threadIdx.x;
  if (p >= n) return;
  const float *q = xyz + ((size_t)b * n + p) * 3;
  float v[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float t = __ldg(q + d);
    if (normalize) {
      // shift_scale_points with dst range [0, 1]: ((x - min) * 1) / (max - min) + 0
      const float lo = __ldg(rmin + b * 3 + d), hi = __ldg(rmax + b * 3 + d);
      t = __fdiv_rn(__fmul_rn(__fsub_rn(t, lo), 1.0f), __fsub_rn(hi, lo)) + 0.0f;
    }
    v[d] = __fmul_rn(t, 6.283185307179586f);  // "xyz *= 2 * np.pi" on an fp32 tensor
  }
  float *o = out + (size_t)b * 2 * d_out * n + p;
  for (int c = 0; c < nc; ++c) {
    const float proj = __fmaf_rn(v[2], sB[2][c], __fmaf_rn(v[1], sB[1][c], __fmul_rn(v[0], sB[0][c])));
    float sn, cs;
    sincosf(proj, &sn, &cs);
    o[(size_t)(c0 + c) * n] = sn;
    o[(size_t)(d_out + c0 + c) * n] = cs;
  }
}

// =====================================================================
//  Generalised 3-D IoU (axis-aligned or rotated-about-up boxes)
// =====================================================================
// P2, sh_inside, sh_intersect, clipped_area: box_geometry.cuh (shared with the evaluation kernels)

__device__ __forceinline__ float edge_len(const float *c, int i, int j) {
  const float dx = c[i * 3] - c[j * 3], dy = c[i * 3 + 1] - c[j * 3 + 1], dz = c[i * 3 + 2] - c[j * 3 + 2];
  return sqrtf(fmaxf(dx * dx + dy * dy + dz * dz, 1e-6f));
}

__global__ void __launch_bounds__(128)
giou3d_kernel(int k1, int k2, int rotated, const int *__restrict__ rotated_dev, int rot_k2_limit,
              const float *__restrict__ corners1, const float *__restrict__ corners2,
              const int *__restrict__ nums_k2, float *__restrict__ gious) {
  if (rotated_dev) rotated = __ldg(rotated_dev) != 0;
  const int b = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= k1 * k2) return;
  const int i = t / k2, j = t % k2;
  float *out = gious + ((size_t)b * k1 + i) * k2 + j;
  const int nk2 = nums_k2 ? __ldg(nums_k2 + b) : k2;
  if (j >= nk2) { *out = 0.f; return; }  // masked columns (box_util.py:751-755)
  float c1[24], c2[24];
  const float *p1 = corners1 + ((size_t)b * k1 + i) * 24;
  const float *p2 = corners2 + ((size_t)b * k2 + j) * 24;
#pragma unroll
  for (int q = 0; q < 24; ++q) { c1[q] = __ldg(p1 + q); c2[q] = __ldg(p2 + q); }
  const float EPS = 1e-8f;
  // height: Y is negative-up (box_util.py:684-686)
  const float ymax = fminf(c1[0 * 3 + 1], c2[0 * 3 + 1]);
  const float ymin = fmaxf(c1[4 * 3 + 1], c2[4 * 3 + 1]);
  const float height = fmaxf(ymax - ymin, 0.f);
  // ground-plane rectangles: corners 3,2,1,0 -> (x, z)   (box_util.py:689-694)
  P2 r1[4], r2[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    r1[q] = P2{c1[(3 - q) * 3 + 0], c1[(3 - q) * 3 + 2]};
    r2[q] = P2{c2[(3 - q) * 3 + 0], c2[(3 - q) * 3 + 2]};
  }
  const float ltx = fmaxf(r1[1].x, r2[1].x), lty = fmaxf(r1[1].y, r2[1].y);
  const float rbx = fminf(r1[3].x, r2[3].x), rby = fminf(r1[3].y, r2[3].y);
  const float non_rot = fmaxf(rbx - ltx, 0.f) * fmaxf(rby - lty, 0.f);
  // enclosing axis-aligned volume (box_util.py:604-652), y flipped
  float xmin = INFINITY, xmax = -INFINITY, zmin = INFINITY, zmax = -INFINITY, fymax = -INFINITY, fymin = INFINITY;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    xmin = fminf(xmin, fminf(c1[q * 3], c2[q * 3]));
    xmax = fmaxf(xmax, fmaxf(c1[q * 3], c2[q * 3]));
    zmin = fminf(zmin, fminf(c1[q * 3 + 2], c2[q * 3 + 2]));
    zmax = fmaxf(zmax, fmaxf(c1[q * 3 + 2], c2[q * 3 + 2]));
    fymax = fmaxf(fymax, fmaxf(-c1[q * 3 + 1], -c2[q * 3 + 1]));  // "al_ymin" = max of flipped y
    fymin = fminf(fymin, fminf(-c1[q * 3 + 1], -c2[q * 3 + 1]));  // "al_ymax" = min of flipped y
  }
  const float enclosing = fabsf(xmax - xmin) * fabsf(fymin - fymax) * fabsf(zmax - zmin);
  const float vol1 = fmaxf(edge_len(c1, 0, 1) * edge_len(c1, 1, 2) * edge_len(c1, 0, 4), EPS);
  const float vol2 = fmaxf(edge_len(c2, 0, 1) * edge_len(c2, 1, 2) * edge_len(c2, 0, 4), EPS);
  const float sum_vols = vol1 + vol2;
  const bool good = (enclosing > 2 * EPS) && (sum_vols > 4 * EPS);
  float inter_area = non_rot;
  if (rotated) {
    inter_area = 0.f;
    if (non_rot != 0.f && j < rot_k2_limit) inter_area = clipped_area(r1, r2);
  }
  const float inter_vol = inter_area * height;
  const float union_vol = fmaxf(sum_vols - inter_vol, EPS);
  const float iou = inter_vol / union_vol;
  const float second = -(1.0f - union_vol / enclosing);
  *out = good ? (iou + second) : 0.f;
}

// =====================================================================
//  Hungarian matching: one warp per scene
// =====================================================================
// Shortest-augmenting-path LSAP exactly as scipy.optimize.linear_sum_assignment
// (scipy/optimize/rectangular_lsap/rectangular_lsap.cpp, Crouse 2016) performs
// it, including its `remaining` ordering and its tie rule, so that ties resolve
// the same way.  The problem is oriented so that rows <= cols ("transpose" when
// there are more proposals than ground-truth boxes): rows = gt, cols = proposals.
struct HungSmem {
  // carved from dynamic shared memory, see hungarian_smem_bytes
  double *u, *v, *spc;
  int *path, *col4row, *row4col, *remaining;
  unsigned char *SR, *SC;
  float *cost;  // nr x nc (row-major), staged when it fits
};

__host__ __device__ inline size_t hungarian_smem_bytes(int nr_max, int nc_max, bool stage_cost) {
  size_t s = 0;
  s += sizeof(double) * (size_t)(nr_max + 2 * nc_max);
  s += sizeof(int) * (size_t)(3 * nc_max + nr_max);
  s += (size_t)(nr_max + nc_max + 15) / 16 * 16;
  if (stage_cost) s += sizeof(float) * (size_t)nr_max * nc_max;
  return s + 64;
}

__global__ void __launch_bounds__(32)
hungarian_kernel(int nprop, int ngt, int stage_cost, const float *__restrict__ cost_all,
                 const int *__restrict__ nactual, long long *__restrict__ per_prop_gt_inds,
                 float *__restrict__ matched_mask) {
  extern __shared__ __align__(16) unsigned char hs[];
  const int lane = threadIdx.x;
  const int b = blockIdx.x;
  const float *cost_g = cost_all + (size_t)b * nprop * ngt;
  long long *gt_out = per_prop_gt_inds + (size_t)b * nprop;
  float *mask_out = matched_mask + (size_t)b * nprop;
  for (int p = lane; p < nprop; p += 32) { gt_out[p] = 0; mask_out[p] = 0.f; }
  int na = __ldg(nactual + b);
  if (na > ngt) na = ngt;
  if (na <= 0) return;
  // orientation: scipy transposes a tall matrix (rows = proposals > cols = gt)
  const bool transposed = na < nprop;
  const int nr = transposed ? na : nprop;
  const int nc = transposed ? nprop : na;
  const int nr_max = min(nprop, ngt) , nc_max = max(nprop, ngt);
  unsigned char *ptr = hs;
  double *u = reinterpret_cast<double *>(ptr); ptr += sizeof(double) * nr_max;
  double *v = reinterpret_cast<double *>(ptr); ptr += sizeof(double) * nc_max;
  double *spc = reinterpret_cast<double *>(ptr); ptr += sizeof(double) * nc_max;
  int *path = reinterpret_cast<int *>(ptr); ptr += sizeof(int) * nc_max;
  int *row4col = reinterpret_cast<int *>(ptr); ptr += sizeof(int) * nc_max;
  int *remaining = reinterpret_cast<int *>(ptr); ptr += sizeof(int) * nc_max;
  int *col4row = reinterpret_cast<int *>(ptr); ptr += sizeof(int) * nr_max;
  unsigned char *SR = ptr; ptr += nr_max;
  unsigned char *SC = ptr; ptr += nc_max;
  ptr = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(ptr) + 15) & ~(uintptr_t)15);
  float *cost_s = reinterpret_cast<float *>(ptr);

  // element (i, j) of the oriented problem
  auto cost_at = [&](int i, int j) -> double {
    if (stage_cost) return (double)cost_s[(size_t)i * nc + j];
    return transposed ? (double)__ldg(cost_g + (size_t)j * ngt + i)
                      : (double)__ldg(cost_g + (size_t)i * ngt + j);
  };
  if (stage_cost) {
    for (int e = lane; e < nr * nc; e += 32) {
      const int i = e / nc, j = e % nc;
      cost_s[e] = transposed ? __ldg(cost_g + (size_t)j * ngt + i) : __ldg(cost_g + (size_t)i * ngt + j);
    }
  }
  for (int i = lane; i < nr; i += 32) { u[i] = 0.0; col4row[i] = -1; }
  for (int j = lane; j < nc; j += 32) { v[j] = 0.0; path[j] = -1; row4col[j] = -1; }
  __syncwarp();

  for (int cur_row = 0; cur_row < nr; ++cur_row) {
    // ---- augmenting_path(cur_row) -------------------------------------
    double min_val = 0.0;
    int num_remaining = nc;
    for (int it = lane; it < nc; it += 32) { remaining[it] = nc - it - 1; spc[it] = INFINITY; SC[it] = 0; }
    for (int i = lane; i < nr; i += 32) SR[i] = 0;
    __syncwarp();
    int sink = -1;
    int i = cur_row;
    while (sink == -1) {
      if (lane == 0) SR[i] = 1;
      const double ui = u[i];
      // each lane scans its positions `it` in ascending order, then lanes are
      // combined so that the result equals scipy's sequential scan:
      //   smallest value; among ties the LAST position with row4col == -1 if any,
      //   otherwise the FIRST position.
      double best = INFINITY;
      int best_it = -1;
      bool best_free = false;
      for (int it = lane; it < num_remaining; it += 32) {
        const int j = remaining[it];
        const double r = min_val + cost_at(i, j) - ui - v[j];
        double sj = spc[j];
        if (r < sj) { path[j] = i; spc[j] = r; sj = r; }
        const bool fr = row4col[j] == -1;
        if (sj < best || (sj == best && fr)) { best = sj; best_it = it; best_free = fr; }
        // within a lane positions ascend, so this is already the sequential rule
      }
      // combine across lanes (positions of different lanes interleave, so apply
      // the rule explicitly on (value, free, it))
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oit = __shfl_xor_sync(0xffffffffu, best_it, o);
        const int ofr = __shfl_xor_sync(0xffffffffu, (int)best_free, o);
        bool take = false;
        if (oit >= 0) {
          if (best_it < 0 || ob < best) take = true;
          else if (ob == best) {
            if (ofr && best_free) take = oit > best_it;        // last free position wins
            else if (ofr && !best_free) take = true;           // a free one beats a non-free one
            else if (!ofr && !best_free) take = oit < best_it; // first position wins
          }
        }
        if (take) { best = ob; best_it = oit; best_free = ofr != 0; }
      }
      // NOTE on the tie rule: sequentially, a non-free tie never replaces the
      // incumbent and a free tie always does; hence "last free if any free exists,
      // else first" -- except that a free incumbent found EARLIER is also replaced by
      // later free ones only, which the rule above reproduces.
      min_val = best;
      if (best_it < 0 || !(min_val < INFINITY)) { sink = -2; break; }  // infeasible
      const int j = remaining[best_it];
      const int r4c = row4col[j];
      if (r4c == -1) sink = j; else i = r4c;
      __syncwarp();
      if (lane == 0) {
        SC[j] = 1;
        remaining[best_it] = remaining[num_remaining - 1];
      }
      --num_remaining;
      __syncwarp();
    }
    if (sink < 0) break;
    // ---- dual update ---------------------------------------------------
    if (lane == 0) u[cur_row] += min_val;
    for (int r = lane; r < nr; r += 32)
      if (SR[r] && r != cur_row) u[r] += min_val - spc[col4row[r]];
    for (int j = lane; j < nc; j += 32)
      if (SC[j]) v[j] -= min_val - spc[j];
    __syncwarp();
    // ---- augment ---------------------------------------------------------
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = r;
        const int t = col4row[r];
        col4row[r] = j;
        j = t;
        if (r == cur_row) break;
      }
    }
    __syncwarp();
  }
  __syncwarp();
  // criterion.py:75-80: per_prop_gt_inds[b, prop] = gt ; proposal_matched_mask[b, prop] = 1
  for (int r = lane; r < nr; r += 32) {
    const int c = col4row[r];
    if (c < 0) continue;
    const int prop = transposed ? c : r, gt = transposed ? r : c;
    gt_out[prop] = gt;
    mask_out[prop] = 1.f;
  }
}

}  // namespace

// =====================================================================
extern "C" {

int coda_layer_norm_fwd_ex(long long rows, int c, float eps, const float *x, const float *gamma,
                           const float *beta, float *y, int y_inner, long long y_so, long long y_si,
                           const float *pos, float *y_pos, float *mean, float *rstd, void *stream) {
  if (rows < 0 || c <= 0 || c % 128 != 0 || c > 1024) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!x || !gamma || !beta || (!y && !y_pos) || ((pos == nullptr) != (y_pos == nullptr))) return CODA_EINVAL;
  if (y_inner < 0 || (y_inner > 0 && ((y_so & 3) || (y_si & 3)))) return CODA_EINVAL;
  const RowMap ymap{y_inner, y_so, y_si};
  const unsigned grid = (unsigned)((rows + LN_WARPS - 1) / LN_WARPS);
  cudaStream_t s = (cudaStream_t)stream;
#define CODA_LN_FWD(NV) \
  case NV: layer_norm_fwd_kernel<NV><<<grid, LN_WARPS * 32, 0, s>>>(rows, eps, x, gamma, beta, y, ymap, pos, y_pos, \
                                                                     mean, rstd); break;
  switch (c / 128) {
    CODA_LN_FWD(1) CODA_LN_FWD(2) CODA_LN_FWD(3) CODA_LN_FWD(4)
    CODA_LN_FWD(5) CODA_LN_FWD(6) CODA_LN_FWD(7) CODA_LN_FWD(8)
  }
#undef CODA_LN_FWD
  return launch_status();
}

int coda_layer_norm_fwd(long long rows, int c, float eps, const float *x, const float *gamma,
                        const float *beta, float *y, float *mean, float *rstd, void *stream) {
  if (!y) return rows == 0 ? CODA_OK : CODA_EINVAL;
  return coda_layer_norm_fwd_ex(rows, c, eps, x, gamma, beta, y, 0, 0, 0, nullptr, nullptr, mean, rstd, stream);
}

int coda_layer_norm_fwd_half(long long rows, int c, float eps, const void *x, const float *gamma,
                             const float *beta, void *y, void *stream) {
  if (rows < 0 || c <= 0 || c % 128 != 0 || c > 1024) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!x || !gamma || !beta || !y) return CODA_EINVAL;
  const unsigned grid = (unsigned)((rows + LN_WARPS - 1) / LN_WARPS);
  cudaStream_t s = (cudaStream_t)stream;
#define CODA_LN_FWD(NV) \
  case NV: layer_norm_fwd_half_kernel<NV><<<grid, LN_WARPS * 32, 0, s>>>( \
      rows, eps, (const __half *)x, gamma, beta, (__half *)y); break;
  switch (c / 128) {
    CODA_LN_FWD(1) CODA_LN_FWD(2) CODA_LN_FWD(3) CODA_LN_FWD(4)
    CODA_LN_FWD(5) CODA_LN_FWD(6) CODA_LN_FWD(7) CODA_LN_FWD(8)
  }
#undef CODA_LN_FWD
  return launch_status();
}

long long coda_layer_norm_bwd_scratch(long long rows, int c) {
  const long long nblk = (rows + LN_BWD_ROWS_PER_BLOCK - 1) / LN_BWD_ROWS_PER_BLOCK;
  return nblk * 2 * c;
}

int coda_layer_norm_bwd_ex(long long rows, int c, const float *dy, int dy_inner, long long dy_so, long long dy_si,
                           const float *dy2, const float *add, const float *x, const float *gamma,
                           const float *mean, const float *rstd, float *dx, float *dgamma,
                           float *dbeta, float *partial, void *stream) {
  if (rows < 0 || c <= 0 || c % 128 != 0 || c > 1024) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  if (rows == 0) {
    if (dgamma) cudaMemsetAsync(dgamma, 0, sizeof(float) * c, s);
    if (dbeta) cudaMemsetAsync(dbeta, 0, sizeof(float) * c, s);
    return launch_status();
  }
  if (!dy || !x || !gamma || !mean || !rstd || !dx || !dgamma || !dbeta || !partial) return CODA_EINVAL;
  if (dy_inner < 0 || (dy_inner > 0 && ((dy_so & 3) || (dy_si & 3)))) return CODA_EINVAL;
  const RowMap dmap{dy_inner, dy_so, dy_si};
  const int nblk = (int)((rows + LN_BWD_ROWS_PER_BLOCK - 1) / LN_BWD_ROWS_PER_BLOCK);
#define CODA_LN_BWD(NV) \
  case NV: layer_norm_bwd_kernel<NV><<<nblk, LN_WARPS * 32, 0, s>>>(rows, dy, dmap, dy2, add, x, gamma, mean, rstd, \
                                                                    dx, partial); break;
  switch (c / 128) {
    CODA_LN_BWD(1) CODA_LN_BWD(2) CODA_LN_BWD(3) CODA_LN_BWD(4)
    CODA_LN_BWD(5) CODA_LN_BWD(6) CODA_LN_BWD(7) CODA_LN_BWD(8)
  }
#undef CODA_LN_BWD
  int st = launch_status();
  if (st != CODA_OK) return st;
  layer_norm_bwd_finalize<<<(2 * c + 255) / 256, 256, 0, s>>>(nblk, c, partial, dgamma, dbeta);
  return launch_status();
}

int coda_layer_norm_bwd(long long rows, int c, const float *dy, const float *x, const float *gamma,
                        const float *mean, const float *rstd, float *dx, float *dgamma,
                        float *dbeta, float *partial, void *stream) {
  return coda_layer_norm_bwd_ex(rows, c, dy, 0, 0, 0, nullptr, nullptr, x, gamma, mean, rstd, dx, dgamma, dbeta,
                                partial, stream);
}

int coda_softmax_rows(long long rows, int c, int log_softmax, const float *x, float *y, void *stream) {
  if (rows < 0 || c <= 0) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!x || !y) return CODA_EINVAL;
  softmax_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(rows, c, log_softmax, x, y);
  return launch_status();
}

int coda_fourier_pos_embed(int b, int n, int d_out, int ldb, int normalize, const float *xyz,
                           const float *range_min, const float *range_max, const float *gauss_b,
                           float *out, void *stream) {
  if (b < 0 || n < 0 || d_out <= 0 || ldb < d_out) return CODA_EINVAL;
  if (b == 0 || n == 0) return CODA_OK;
  if (!xyz || !gauss_b || !out || (normalize && (!range_min || !range_max)) || b > 65535) return CODA_EINVAL;
  const dim3 grid((n + 127) / 128, (d_out + FOURIER_CH - 1) / FOURIER_CH, b);
  fourier_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(n, d_out, ldb, normalize, xyz, range_min,
                                                        range_max, gauss_b, out);
  return launch_status();
}

int coda_giou3d(int b, int k1, int k2, int rotated, const int *rotated_dev, int rot_k2_limit,
                const float *corners1, const float *corners2, const int *nums_k2, float *gious,
                void *stream) {
  if (b < 0 || k1 < 0 || k2 < 0) return CODA_EINVAL;
  if (b == 0 || k1 == 0 || k2 == 0) return CODA_OK;
  if (!corners1 || !corners2 || !gious || b > 65535) return CODA_EINVAL;
  const dim3 grid((k1 * k2 + 127) / 128, b);
  giou3d_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(k1, k2, rotated, rotated_dev, rot_k2_limit, corners1,
                                                       corners2, nums_k2, gious);
  return launch_status();
}

int coda_hungarian(int b, int nprop, int ngt, const float *cost, const int *nactual,
                   long long *per_prop_gt_inds, float *proposal_matched_mask, void *stream) {
  if (b < 0 || nprop < 0 || ngt < 0) return CODA_EINVAL;
  if (b == 0 || nprop == 0) return CODA_OK;
  if (!nactual || !per_prop_gt_inds || !proposal_matched_mask || (ngt > 0 && !cost)) return CODA_EINVAL;
  if (ngt == 0) {
    cudaMemsetAsync(per_prop_gt_inds, 0, sizeof(long long) * (size_t)b * nprop, (cudaStream_t)stream);
    cudaMemsetAsync(proposal_matched_mask, 0, sizeof(float) * (size_t)b * nprop, (cudaStream_t)stream);
    return launch_status();
  }
  const int nr_max = nprop < ngt ? nprop : ngt, nc_max = nprop < ngt ? ngt : nprop;
  int stage = 1;
  size_t smem = hungarian_smem_bytes(nr_max, nc_max, true);
  if (smem > 200 * 1024) { stage = 0; smem = hungarian_smem_bytes(nr_max, nc_max, false); }
  if (smem > 200 * 1024) return CODA_ETOOLARGE;
  cudaError_t e = cudaFuncSetAttribute(hungarian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  hungarian_kernel<<<b, 32, smem, (cudaStream_t)stream>>>(nprop, ngt, stage, cost, nactual, per_prop_gt_inds,
                                                         proposal_matched_mask);
  return launch_status();
}

}  // extern "C"
