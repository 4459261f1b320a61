// Row-streaming kernels of the PointNet++ shared MLP for H100 (sm_90a): everything that sits between two
// tensor-core GEMMs of Conv1x1 -> BatchNorm -> ReLU blocks, one HBM pass each.  C-ABI in include/coda_sa_mlp.h.
//
// These kernels are HBM-bound by construction (a (1M, 256) fp32 activation is 1 GB): the design rule is to
// touch every activation once per direction.  Layout: channels-last rows; a thread owns FOUR channels
// (one float4 per row) for the whole kernel, c/4 threads span a row, 256/(c/4) rows are in flight per block
// iteration, blocks grid-stride over rows.  Per-channel parameters therefore live in registers, row loads are
// 16-byte and fully coalesced, and every column reduction is thread-local until one smem pass at the end.
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>

#include "../../include/coda_sa_mlp.h"
#include "coda_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int MAX_BLOCKS = 132 * 4;   // persistent-style grid: 4 resident blocks per SM of an H100 SXM

__host__ __device__ inline bool channels_ok(int c) { return c >= 4 && c <= 1024 && c % 4 == 0 && THREADS % (c / 4) == 0; }

__host__ inline unsigned grid_for(long long rows, int c) {
  const long long per_iter = THREADS / (c / 4);
  const long long need = (rows + per_iter - 1) / per_iter;
  return (unsigned)(need < MAX_BLOCKS ? (need > 0 ? need : 1) : MAX_BLOCKS);
}

struct Affine4 {
  float4 mean, invstd, gamma, beta;
};
__device__ __forceinline__ Affine4 load_affine(const float *mean, const float *invstd, const float *gamma,
                                               const float *beta, int c4) {
  Affine4 a;
  a.mean = __ldg(reinterpret_cast<const float4 *>(mean) + c4);
  a.invstd = __ldg(reinterpret_cast<const float4 *>(invstd) + c4);
  a.gamma = __ldg(reinterpret_cast<const float4 *>(gamma) + c4);
  a.beta = __ldg(reinterpret_cast<const float4 *>(beta) + c4);
  return a;
}
__device__ __forceinline__ float4 xhat4(const float4 v, const Affine4 &a) {
  return make_float4((v.x - a.mean.x) * a.invstd.x, (v.y - a.mean.y) * a.invstd.y, (v.z - a.mean.z) * a.invstd.z,
                     (v.w - a.mean.w) * a.invstd.w);
}
__device__ __forceinline__ float4 bn4(const float4 xh, const Affine4 &a) {
  return make_float4(xh.x * a.gamma.x + a.beta.x, xh.y * a.gamma.y + a.beta.y, xh.z * a.gamma.z + a.beta.z,
                     xh.w * a.gamma.w + a.beta.w);
}

// four values -> NS bf16 planes, 8 bytes per plane
template <int NS>
__device__ __forceinline__ void store_planes4(float4 v, __nv_bfloat16 *dst, size_t plane_stride) {
  float r[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int p = 0; p < NS; ++p) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(r[0], r[1]), hi = __floats2bfloat162_rn(r[2], r[3]);
    uint2 w;
    w.x = *reinterpret_cast<const uint32_t *>(&lo);
    w.y = *reinterpret_cast<const uint32_t *>(&hi);
    *reinterpret_cast<uint2 *>(dst + (size_t)p * plane_stride) = w;
    if (p + 1 < NS) {
      r[0] -= __uint_as_float(w.x << 16); r[1] -= __uint_as_float(w.x & 0xFFFF0000u);
      r[2] -= __uint_as_float(w.y << 16); r[3] -= __uint_as_float(w.y & 0xFFFF0000u);
    }
  }
}

// block-level sum of NV float4 accumulators over the row slots; thread (slot 0, c4) ends with the total
template <int NV>
__device__ __forceinline__ void reduce_slots(float4 (&acc)[NV], int cq, int slot, int c4, float4 *red /*[THREADS]*/) {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    __syncthreads();
    red[threadIdx.x] = acc[i];
    __syncthreads();
    if (slot == 0) {
      float4 t = acc[i];
      for (int s = 1; s < THREADS / cq; ++s) {
        const float4 o = red[s * cq + c4];
        t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w;
      }
      acc[i] = t;
    }
  }
}

// ------------------------------------------------------------------ first layer: tiny-K linear
template <int CIN>
__global__ void __launch_bounds__(THREADS)
linear_small_k_kernel(long long rows, int cout, const float *__restrict__ x, const float *__restrict__ w,
                      float *__restrict__ y) {
  const int cq = cout >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  float wr[4][CIN];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < CIN; ++k) wr[j][k] = __ldg(w + (size_t)(c4 * 4 + j) * CIN + k);
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    float xv[CIN];
#pragma unroll
    for (int k = 0; k < CIN; ++k) xv[k] = __ldg(x + r * CIN + k);
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = xv[0] * wr[j][0];
#pragma unroll
      for (int k = 1; k < CIN; ++k) a = fmaf(xv[k], wr[j][k], a);
      o[j] = a;
    }
    reinterpret_cast<float4 *>(y + r * cout)[c4] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------ statistics
// partial[blk][0][c] = sum, partial[blk][1][c] = sum of squares over the block's rows
__global__ void __launch_bounds__(THREADS)
bn_stats_partial_kernel(long long rows, int c, const float *__restrict__ y, float *__restrict__ partial) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  float4 acc[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 v = __ldg(reinterpret_cast<const float4 *>(y + r * c) + c4);
    acc[0].x += v.x; acc[0].y += v.y; acc[0].z += v.z; acc[0].w += v.w;
    acc[1].x = fmaf(v.x, v.x, acc[1].x); acc[1].y = fmaf(v.y, v.y, acc[1].y);
    acc[1].z = fmaf(v.z, v.z, acc[1].z); acc[1].w = fmaf(v.w, v.w, acc[1].w);
  }
  reduce_slots<2>(acc, cq, slot, c4, red);
  if (slot == 0) {
    float4 *p = reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * 2 * c);
    p[c4] = acc[0];
    p[cq + c4] = acc[1];
  }
}
// one WARP per channel: lanes stride over the block partials (fp64), then a shuffle tree
__device__ __forceinline__ void warp_partials_sum(int nblocks, int c, int ch, const float *__restrict__ partial,
                                                  double &s, double &q) {
  const int lane = threadIdx.x & 31;
  s = 0.0; q = 0.0;
  for (int b = lane; b < nblocks; b += 32) {
    s += (double)partial[(size_t)b * 2 * c + ch];
    q += (double)partial[(size_t)b * 2 * c + c + ch];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
}
__global__ void __launch_bounds__(256)
bn_stats_finalize_kernel(int nblocks, long long rows, int c, const float *__restrict__ partial,
                         float eps, float momentum, float *running_mean, float *running_var,
                         float *__restrict__ mean, float *__restrict__ invstd) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (ch >= c) return;
  double s, q;
  warp_partials_sum(nblocks, c, ch, partial, s, q);
  if ((threadIdx.x & 31) != 0) return;
  const double n = (double)rows, m = s / n;
  double var = q / n - m * m;
  if (var < 0.0) var = 0.0;
  mean[ch] = (float)m;
  invstd[ch] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean) running_mean[ch] = (1.0f - momentum) * running_mean[ch] + momentum * (float)m;
  if (running_var) running_var[ch] = (1.0f - momentum) * running_var[ch] + momentum * (float)(var * (n / fmax(n - 1.0, 1.0)));
}

// finalisation of per-CTA partials written by a GEMM epilogue (coda_gemm_a32 col_stats): statistics + running
// buffers as above, plus the folded per-channel affine map of BatchNorm: scale = gamma * invstd,
// shift = beta - mean * scale (what the next GEMM's prologue applies), zero-padded up to cpad
__global__ void __launch_bounds__(256)
bn_stats_finalize_affine_kernel(int nblocks, long long rows, int c, int cpad,
                                                const float *__restrict__ partial, float eps, float momentum,
                                                float *running_mean, float *running_var, const float *__restrict__ gamma,
                                                const float *__restrict__ beta, float *__restrict__ mean,
                                                float *__restrict__ invstd, float *__restrict__ scale,
                                                float *__restrict__ shift) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (ch >= cpad) return;
  if (ch >= c) {
    if (scale && (threadIdx.x & 31) == 0) { scale[ch] = 0.f; shift[ch] = 0.f; }
    return;
  }
  double s, q;
  warp_partials_sum(nblocks, c, ch, partial, s, q);
  if ((threadIdx.x & 31) != 0) return;
  const double n = (double)rows, m = s / n;
  double var = q / n - m * m;
  if (var < 0.0) var = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[ch] = (float)m;
  invstd[ch] = is;
  if (running_mean) running_mean[ch] = (1.0f - momentum) * running_mean[ch] + momentum * (float)m;
  if (running_var) running_var[ch] = (1.0f - momentum) * running_var[ch] + momentum * (float)(var * (n / fmax(n - 1.0, 1.0)));
  if (scale) {
    const float sc = gamma[ch] * is;
    scale[ch] = sc;
    shift[ch] = beta[ch] - (float)m * sc;
  }
}
// ---- synchronised BatchNorm (statistics over the batches of ALL ranks, reference main.py:993 convert_sync_batchnorm)
// Stage 1 on each rank: the per-channel column sums as fp64 [sum(c) | sum of squares(c)] -- what the ranks
// all-reduce (fp64: E[x^2] - E[x]^2 from fp32 sums would cancel catastrophically for |mean| >> std).
__global__ void __launch_bounds__(256)
bn_sums_f64_kernel(int nblocks, int c, const float *__restrict__ partial, double *__restrict__ sums) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (ch >= c) return;
  double s, q;
  warp_partials_sum(nblocks, c, ch, partial, s, q);
  if ((threadIdx.x & 31) != 0) return;
  sums[ch] = s;
  sums[c + ch] = q;
}
// Stage 2 (after the all-reduce): statistics over `rows` = the global row count, running buffers, folded affine map
__global__ void __launch_bounds__(256)
bn_finalize_sums_kernel(long long rows, int c, int cpad, const double *__restrict__ sums, float eps, float momentum,
                        float *running_mean, float *running_var, const float *__restrict__ gamma,
                        const float *__restrict__ beta, float *__restrict__ mean, float *__restrict__ invstd,
                        float *__restrict__ scale, float *__restrict__ shift) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= cpad) return;
  if (ch >= c) {
    if (scale) { scale[ch] = 0.f; shift[ch] = 0.f; }
    return;
  }
  const double n = (double)rows, m = sums[ch] / n;
  double var = sums[c + ch] / n - m * m;
  if (var < 0.0) var = 0.0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[ch] = (float)m;
  invstd[ch] = is;
  if (running_mean) running_mean[ch] = (1.0f - momentum) * running_mean[ch] + momentum * (float)m;
  if (running_var) running_var[ch] = (1.0f - momentum) * running_var[ch] + momentum * (float)(var * (n / fmax(n - 1.0, 1.0)));
  if (scale) {
    const float sc = gamma[ch] * is;
    scale[ch] = sc;
    shift[ch] = beta[ch] - (float)m * sc;
  }
}

// BatchNorm-backward coefficients of the GEMM prologue: dy = [z > 0] * scale * d + alpha * y + beta
//   alpha = -scale * invstd * s2 / N,   beta = -scale * s1 / N - alpha * mean
__global__ void bn_bwd_coefs_kernel(int c, int cpad, long long rows, const float *__restrict__ mean,
                                    const float *__restrict__ invstd, const float *__restrict__ gamma,
                                    const float *__restrict__ s1, const float *__restrict__ s2,
                                    float *__restrict__ alpha, float *__restrict__ beta) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= cpad) return;
  if (ch >= c) { alpha[ch] = 0.f; beta[ch] = 0.f; return; }
  const float inv_n = 1.0f / (float)rows;
  const float sc = gamma[ch] * invstd[ch];
  const float a = -sc * invstd[ch] * (s2[ch] * inv_n);
  alpha[ch] = a;
  beta[ch] = -sc * (s1[ch] * inv_n) - a * mean[ch];
}

// column sums only (bias gradients: db = sum over rows of dY); partial[blk][c]
__global__ void __launch_bounds__(THREADS)
colsum_partial_kernel(long long rows, int c, const float *__restrict__ x, float *__restrict__ partial) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  float4 acc[1] = {make_float4(0.f, 0.f, 0.f, 0.f)};
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 v = __ldg(reinterpret_cast<const float4 *>(x + r * c) + c4);
    acc[0].x += v.x; acc[0].y += v.y; acc[0].z += v.z; acc[0].w += v.w;
  }
  reduce_slots<1>(acc, cq, slot, c4, red);
  if (slot == 0) reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * c)[c4] = acc[0];
}
// one warp per channel: lanes stride over the block partials, then a shuffle tree
__global__ void __launch_bounds__(256)
colsum_finalize_kernel(int nblocks, int c, const float *__restrict__ partial, float *__restrict__ out) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (ch >= c) return;
  float a = 0.f;
  for (int k = lane; k < nblocks; k += 32) a += partial[(size_t)k * c + ch];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) out[ch] = a;
}

// ------------------------------------------------------------------ forward: normalise + ReLU + operand planes
template <int NS>
__global__ void __launch_bounds__(THREADS)
bn_relu_pack_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ mean,
                    const float *__restrict__ invstd, const float *__restrict__ gamma, const float *__restrict__ beta,
                    __nv_bfloat16 *__restrict__ planes) {
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const size_t plane_stride = (size_t)rows * c;
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 z = bn4(xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a), a);
    store_planes4<NS>(make_float4(fmaxf(z.x, 0.f), fmaxf(z.y, 0.f), fmaxf(z.z, 0.f), fmaxf(z.w, 0.f)),
                      planes + r * c + c4 * 4, plane_stride);
  }
}

// one block iteration = one group of `group` rows; slots split the group's rows, smem merges them
__global__ void __launch_bounds__(THREADS)
bn_relu_maxpool_kernel(long long groups, int group, int c, const float *__restrict__ y, const float *__restrict__ mean,
                       const float *__restrict__ invstd, const float *__restrict__ gamma,
                       const float *__restrict__ beta, float *__restrict__ pooled, unsigned char *__restrict__ argmax) {
  __shared__ float4 sval[THREADS];
  __shared__ uchar4 sidx[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uchar4 bi = make_uchar4(0, 0, 0, 0);
    for (int i = slot; i < group; i += nslots) {
      const float4 zz = bn4(xhat4(__ldg(reinterpret_cast<const float4 *>(y + (g * group + i) * c) + c4), a), a);
      const float4 z = make_float4(fmaxf(zz.x, 0.f), fmaxf(zz.y, 0.f), fmaxf(zz.z, 0.f), fmaxf(zz.w, 0.f));
      if (z.x > best.x) { best.x = z.x; bi.x = (unsigned char)i; }
      if (z.y > best.y) { best.y = z.y; bi.y = (unsigned char)i; }
      if (z.z > best.z) { best.z = z.z; bi.z = (unsigned char)i; }
      if (z.w > best.w) { best.w = z.w; bi.w = (unsigned char)i; }
    }
    __syncthreads();   // (previous iteration's readers are done)
    sval[threadIdx.x] = best;
    sidx[threadIdx.x] = bi;
    __syncthreads();
    if (slot == 0) {
      for (int s = 1; s < nslots; ++s) {
        const float4 o = sval[s * cq + c4];
        const uchar4 oi = sidx[s * cq + c4];
        // first maximum wins (F.max_pool2d): strictly greater, or equal with a smaller row index
        if (o.x > best.x || (o.x == best.x && oi.x < bi.x)) { best.x = o.x; bi.x = oi.x; }
        if (o.y > best.y || (o.y == best.y && oi.y < bi.y)) { best.y = o.y; bi.y = oi.y; }
        if (o.z > best.z || (o.z == best.z && oi.z < bi.z)) { best.z = o.z; bi.z = oi.z; }
        if (o.w > best.w || (o.w == best.w && oi.w < bi.w)) { best.w = o.w; bi.w = oi.w; }
      }
      reinterpret_cast<float4 *>(pooled + g * c)[c4] = best;
      reinterpret_cast<uchar4 *>(argmax + g * c)[c4] = bi;
    }
  }
}

// ------------------------------------------------------------------ backward, first half: dbeta / dgamma sums
__global__ void __launch_bounds__(THREADS)
bn_relu_bwd_reduce_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ dz,
                          const float *__restrict__ mean, const float *__restrict__ invstd,
                          const float *__restrict__ gamma, const float *__restrict__ beta, float *__restrict__ partial) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  float4 acc[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 xh = xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a);
    const float4 z = bn4(xh, a);
    float4 d = __ldg(reinterpret_cast<const float4 *>(dz + r * c) + c4);
    d.x = z.x > 0.f ? d.x : 0.f; d.y = z.y > 0.f ? d.y : 0.f; d.z = z.z > 0.f ? d.z : 0.f; d.w = z.w > 0.f ? d.w : 0.f;
    acc[0].x += d.x; acc[0].y += d.y; acc[0].z += d.z; acc[0].w += d.w;
    acc[1].x = fmaf(d.x, xh.x, acc[1].x); acc[1].y = fmaf(d.y, xh.y, acc[1].y);
    acc[1].z = fmaf(d.z, xh.z, acc[1].z); acc[1].w = fmaf(d.w, xh.w, acc[1].w);
  }
  reduce_slots<2>(acc, cq, slot, c4, red);
  if (slot == 0) {
    float4 *p = reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * 2 * c);
    p[c4] = acc[0];
    p[cq + c4] = acc[1];
  }
}
// pooled form: only the arg-max row of each (group, channel) carries a gradient
__global__ void __launch_bounds__(THREADS)
bn_relu_bwd_reduce_pooled_kernel(long long groups, int group, int c, const float *__restrict__ y,
                                 const float *__restrict__ dpooled, const unsigned char *__restrict__ argmax,
                                 const float *__restrict__ mean, const float *__restrict__ invstd,
                                 const float *__restrict__ gamma, const float *__restrict__ beta,
                                 float *__restrict__ partial, float *__restrict__ dprime) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  float4 acc[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  for (long long g = (long long)blockIdx.x * nslots + slot; g < groups; g += (long long)gridDim.x * nslots) {
    const uchar4 id = __ldg(reinterpret_cast<const uchar4 *>(argmax + g * c) + c4);
    const float *base = y + g * group * c + c4 * 4;
    const float4 v = make_float4(__ldg(base + (size_t)id.x * c), __ldg(base + (size_t)id.y * c + 1),
                                 __ldg(base + (size_t)id.z * c + 2), __ldg(base + (size_t)id.w * c + 3));
    const float4 xh = xhat4(v, a);
    const float4 z = bn4(xh, a);
    float4 d = __ldg(reinterpret_cast<const float4 *>(dpooled + g * c) + c4);
    d.x = z.x > 0.f ? d.x : 0.f; d.y = z.y > 0.f ? d.y : 0.f; d.z = z.z > 0.f ? d.z : 0.f; d.w = z.w > 0.f ? d.w : 0.f;
    if (dprime)      // masked gradient times gamma * invstd: what the GEMM prologues add at the arg-max row
      reinterpret_cast<float4 *>(dprime + g * c)[c4] =
          make_float4(a.gamma.x * a.invstd.x * d.x, a.gamma.y * a.invstd.y * d.y, a.gamma.z * a.invstd.z * d.z,
                      a.gamma.w * a.invstd.w * d.w);
    acc[0].x += d.x; acc[0].y += d.y; acc[0].z += d.z; acc[0].w += d.w;
    acc[1].x = fmaf(d.x, xh.x, acc[1].x); acc[1].y = fmaf(d.y, xh.y, acc[1].y);
    acc[1].z = fmaf(d.z, xh.z, acc[1].z); acc[1].w = fmaf(d.w, xh.w, acc[1].w);
  }
  reduce_slots<2>(acc, cq, slot, c4, red);
  if (slot == 0) {
    float4 *p = reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * 2 * c);
    p[c4] = acc[0];
    p[cq + c4] = acc[1];
  }
}
__global__ void __launch_bounds__(256)
sums_finalize_kernel(int nblocks, int c, const float *__restrict__ partial, float *__restrict__ s1,
                     float *__restrict__ s2) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (ch >= c) return;
  double a, b;
  warp_partials_sum(nblocks, c, ch, partial, a, b);
  if ((threadIdx.x & 31) == 0) {
    s1[ch] = (float)a;
    s2[ch] = (float)b;
  }
}

// ------------------------------------------------------------------ backward, second half
// dy = gamma * invstd * (dz_masked - s1 / N - xhat * s2 / N)
struct BwdCoef4 {
  float4 k, m1, m2;   // k = gamma * invstd, m1 = s1 / N, m2 = s2 / N
};
__device__ __forceinline__ BwdCoef4 load_coef(const Affine4 &a, const float *s1, const float *s2, int c4, float inv_n) {
  const float4 t1 = __ldg(reinterpret_cast<const float4 *>(s1) + c4), t2 = __ldg(reinterpret_cast<const float4 *>(s2) + c4);
  BwdCoef4 q;
  q.k = make_float4(a.gamma.x * a.invstd.x, a.gamma.y * a.invstd.y, a.gamma.z * a.invstd.z, a.gamma.w * a.invstd.w);
  q.m1 = make_float4(t1.x * inv_n, t1.y * inv_n, t1.z * inv_n, t1.w * inv_n);
  q.m2 = make_float4(t2.x * inv_n, t2.y * inv_n, t2.z * inv_n, t2.w * inv_n);
  return q;
}
__device__ __forceinline__ float4 dy4(const float4 d, const float4 xh, const BwdCoef4 &q) {
  return make_float4(q.k.x * (d.x - q.m1.x - xh.x * q.m2.x), q.k.y * (d.y - q.m1.y - xh.y * q.m2.y),
                     q.k.z * (d.z - q.m1.z - xh.z * q.m2.z), q.k.w * (d.w - q.m1.w - xh.w * q.m2.w));
}

template <int NS, bool POOLED>
__global__ void __launch_bounds__(THREADS)
bn_relu_bwd_pack_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ dz,
                        const float *__restrict__ dpooled, const unsigned char *__restrict__ argmax, int group,
                        const float *__restrict__ mean, const float *__restrict__ invstd,
                        const float *__restrict__ gamma, const float *__restrict__ beta, const float *__restrict__ s1,
                        const float *__restrict__ s2, __nv_bfloat16 *__restrict__ planes) {
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const BwdCoef4 q = load_coef(a, s1, s2, c4, 1.0f / (float)rows);
  const size_t plane_stride = (size_t)rows * c;
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 xh = xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a);
    const float4 z = bn4(xh, a);
    float4 d;
    if (POOLED) {
      const long long g = r / group;
      const int i = (int)(r - g * group);
      const uchar4 id = __ldg(reinterpret_cast<const uchar4 *>(argmax + g * c) + c4);
      const float4 dp = __ldg(reinterpret_cast<const float4 *>(dpooled + g * c) + c4);
      d = make_float4(id.x == i ? dp.x : 0.f, id.y == i ? dp.y : 0.f, id.z == i ? dp.z : 0.f, id.w == i ? dp.w : 0.f);
    } else {
      d = __ldg(reinterpret_cast<const float4 *>(dz + r * c) + c4);
    }
    d.x = z.x > 0.f ? d.x : 0.f; d.y = z.y > 0.f ? d.y : 0.f; d.z = z.z > 0.f ? d.z : 0.f; d.w = z.w > 0.f ? d.w : 0.f;
    store_planes4<NS>(dy4(d, xh, q), planes + r * c + c4 * 4, plane_stride);
  }
}

// first layer: dw[c][k] = sum_r dy[r][c] * x[r][k]; partial[blk][c][k]
template <int CIN>
__global__ void __launch_bounds__(THREADS)
bn_relu_bwd_small_k_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ dz,
                           const float *__restrict__ mean, const float *__restrict__ invstd,
                           const float *__restrict__ gamma, const float *__restrict__ beta,
                           const float *__restrict__ s1, const float *__restrict__ s2, const float *__restrict__ x,
                           float *__restrict__ partial) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const BwdCoef4 q = load_coef(a, s1, s2, c4, 1.0f / (float)rows);
  float4 acc[CIN];
#pragma unroll
  for (int k = 0; k < CIN; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 xh = xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a);
    const float4 z = bn4(xh, a);
    float4 d = __ldg(reinterpret_cast<const float4 *>(dz + r * c) + c4);
    d.x = z.x > 0.f ? d.x : 0.f; d.y = z.y > 0.f ? d.y : 0.f; d.z = z.z > 0.f ? d.z : 0.f; d.w = z.w > 0.f ? d.w : 0.f;
    const float4 g = dy4(d, xh, q);
#pragma unroll
    for (int k = 0; k < CIN; ++k) {
      const float xv = __ldg(x + r * CIN + k);
      acc[k].x = fmaf(g.x, xv, acc[k].x); acc[k].y = fmaf(g.y, xv, acc[k].y);
      acc[k].z = fmaf(g.z, xv, acc[k].z); acc[k].w = fmaf(g.w, xv, acc[k].w);
    }
  }
  reduce_slots<CIN>(acc, cq, slot, c4, red);
  if (slot == 0) {
    float *p = partial + (size_t)blockIdx.x * c * CIN;
#pragma unroll
    for (int k = 0; k < CIN; ++k) {
      p[(size_t)(c4 * 4 + 0) * CIN + k] = acc[k].x;
      p[(size_t)(c4 * 4 + 1) * CIN + k] = acc[k].y;
      p[(size_t)(c4 * 4 + 2) * CIN + k] = acc[k].z;
      p[(size_t)(c4 * 4 + 3) * CIN + k] = acc[k].w;
    }
  }
}
__global__ void dw_finalize_kernel(int nblocks, int n, const float *__restrict__ partial, float *__restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a = 0.0;
  for (int k = 0; k < nblocks; ++k) a += (double)partial[(size_t)k * n + i];
  dw[i] = (float)a;
}

}  // namespace

extern "C" {

long long coda_bn_rows_scratch_floats(int c) { return (long long)MAX_BLOCKS * 2 * c; }
long long coda_bn_rows_small_k_scratch_floats(int cin, int cout) { return (long long)MAX_BLOCKS * cin * cout; }

int coda_rows_linear_small_k(long long rows, int cin, int cout, const float *x, const float *w, float *y,
                             void *stream) {
  if (rows < 0 || cin < 1 || cin > 8 || !channels_ok(cout)) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!x || !w || !y) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, cout);
#define CODA_CASE(K) case K: linear_small_k_kernel<K><<<grid, THREADS, 0, s>>>(rows, cout, x, w, y); break;
  switch (cin) { CODA_CASE(1) CODA_CASE(2) CODA_CASE(3) CODA_CASE(4) CODA_CASE(5) CODA_CASE(6) CODA_CASE(7) CODA_CASE(8) }
#undef CODA_CASE
  return coda::launch_status();
}

int coda_bn_rows_stats(long long rows, int c, const float *y, float eps, float momentum, float *running_mean,
                       float *running_var, float *mean, float *invstd, float *scratch, void *stream) {
  if (rows <= 0 || !channels_ok(c) || !y || !mean || !invstd || !scratch) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  bn_stats_partial_kernel<<<grid, THREADS, 0, s>>>(rows, c, y, scratch);
  bn_stats_finalize_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, rows, c, scratch, eps, momentum, running_mean,
                                                           running_var, mean, invstd);
  return coda::launch_status();
}

int coda_bn_rows_stats_affine(long long rows, int c, const float *y, float eps, float momentum, float *running_mean,
                               float *running_var, const float *gamma, const float *beta, float *mean, float *invstd,
                               float *scale, float *shift, float *scratch, void *stream) {
  if (rows <= 0 || !channels_ok(c) || !y || !mean || !invstd || !scratch || !gamma || !beta || !scale || !shift)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  bn_stats_partial_kernel<<<grid, THREADS, 0, s>>>(rows, c, y, scratch);
  const int cpad = (c + 63) / 64 * 64;
  bn_stats_finalize_affine_kernel<<<(cpad + 7) / 8, 256, 0, s>>>((int)grid, rows, c, cpad, scratch, eps, momentum,
                                                                    running_mean, running_var, gamma, beta, mean,
                                                                    invstd, scale, shift);
  return coda::launch_status();
}

int coda_bn_stats_finalize(int nblocks, long long rows, int c, const float *partial, float eps, float momentum,
                           float *running_mean, float *running_var, const float *gamma, const float *beta,
                           float *mean, float *invstd, float *scale, float *shift, void *stream) {
  if (nblocks <= 0 || rows <= 0 || c <= 0 || !partial || !mean || !invstd) return CODA_EINVAL;
  if ((scale != nullptr) != (shift != nullptr) || (scale && (!gamma || !beta))) return CODA_EINVAL;
  const int cpad = (c + 63) / 64 * 64;
  bn_stats_finalize_affine_kernel<<<(cpad + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
      nblocks, rows, c, cpad, partial, eps, momentum, running_mean, running_var, gamma, beta, mean, invstd, scale, shift);
  return coda::launch_status();
}

int coda_bn_rows_sums(long long rows, int c, const float *y, double *sums, float *scratch, void *stream) {
  if (rows <= 0 || !channels_ok(c) || !y || !sums || !scratch) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  bn_stats_partial_kernel<<<grid, THREADS, 0, s>>>(rows, c, y, scratch);
  bn_sums_f64_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, c, scratch, sums);
  return coda::launch_status();
}

int coda_bn_partials_sums(int nblocks, int c, const float *partial, double *sums, void *stream) {
  if (nblocks <= 0 || c <= 0 || !partial || !sums) return CODA_EINVAL;
  bn_sums_f64_kernel<<<(c + 7) / 8, 256, 0, (cudaStream_t)stream>>>(nblocks, c, partial, sums);
  return coda::launch_status();
}

int coda_bn_stats_finalize_sums(long long rows, int c, const double *sums, float eps, float momentum,
                                float *running_mean, float *running_var, const float *gamma, const float *beta,
                                float *mean, float *invstd, float *scale, float *shift, void *stream) {
  if (rows <= 0 || c <= 0 || !sums || !mean || !invstd) return CODA_EINVAL;
  if ((scale != nullptr) != (shift != nullptr) || (scale && (!gamma || !beta))) return CODA_EINVAL;
  const int cpad = scale ? (c + 63) / 64 * 64 : c;
  bn_finalize_sums_kernel<<<(cpad + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      rows, c, cpad, sums, eps, momentum, running_mean, running_var, gamma, beta, mean, invstd, scale, shift);
  return coda::launch_status();
}

int coda_bn_bwd_coefs(int c, long long rows, const float *mean, const float *invstd, const float *gamma,
                      const float *s1, const float *s2, float *alpha, float *beta, void *stream) {
  if (c <= 0 || rows <= 0 || !mean || !invstd || !gamma || !s1 || !s2 || !alpha || !beta) return CODA_EINVAL;
  const int cpad = (c + 63) / 64 * 64;
  bn_bwd_coefs_kernel<<<(cpad + 127) / 128, 128, 0, (cudaStream_t)stream>>>(c, cpad, rows, mean, invstd, gamma, s1, s2,
                                                                           alpha, beta);
  return coda::launch_status();
}

int coda_rows_colsum(long long rows, int c, const float *x, float *out, float *scratch, void *stream) {
  if (rows <= 0 || !channels_ok(c) || !x || !out || !scratch) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  // short matrices: fewer blocks keep the second stage short
  unsigned grid = grid_for(rows, c);
  if (grid > 132) grid = 132;
  colsum_partial_kernel<<<grid, THREADS, 0, s>>>(rows, c, x, scratch);
  colsum_finalize_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, c, scratch, out);
  return coda::launch_status();
}

int coda_bn_relu_pack_rows(long long rows, int c, int nsplit, const float *y, const float *mean,
                           const float *invstd, const float *gamma, const float *beta, void *planes,
                           void *stream) {
  if (rows < 0 || !channels_ok(c) || c % 64 != 0 || nsplit < 1 || nsplit > 3) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!y || !mean || !invstd || !gamma || !beta || !planes) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  __nv_bfloat16 *p = (__nv_bfloat16 *)planes;
  if (nsplit == 1) bn_relu_pack_kernel<1><<<grid, THREADS, 0, s>>>(rows, c, y, mean, invstd, gamma, beta, p);
  else if (nsplit == 2) bn_relu_pack_kernel<2><<<grid, THREADS, 0, s>>>(rows, c, y, mean, invstd, gamma, beta, p);
  else bn_relu_pack_kernel<3><<<grid, THREADS, 0, s>>>(rows, c, y, mean, invstd, gamma, beta, p);
  return coda::launch_status();
}

int coda_bn_relu_maxpool_rows(long long groups, int group, int c, const float *y, const float *mean,
                              const float *invstd, const float *gamma, const float *beta, float *pooled,
                              unsigned char *argmax, void *stream) {
  if (groups < 0 || group < 1 || group > 256 || !channels_ok(c)) return CODA_EINVAL;
  if (groups == 0) return CODA_OK;
  if (!y || !mean || !invstd || !gamma || !beta || !pooled || !argmax) return CODA_EINVAL;
  const unsigned grid = (unsigned)(groups < 132 * 8 ? groups : 132 * 8);
  bn_relu_maxpool_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(groups, group, c, y, mean, invstd, gamma, beta,
                                                                    pooled, argmax);
  return coda::launch_status();
}

int coda_bn_relu_bwd_reduce(long long rows, int c, const float *y, const float *dz, const float *mean,
                            const float *invstd, const float *gamma, const float *beta, float *s1, float *s2,
                            float *scratch, void *stream) {
  if (rows <= 0 || !channels_ok(c) || !y || !dz || !mean || !invstd || !gamma || !beta || !s1 || !s2 || !scratch)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  bn_relu_bwd_reduce_kernel<<<grid, THREADS, 0, s>>>(rows, c, y, dz, mean, invstd, gamma, beta, scratch);
  sums_finalize_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, c, scratch, s1, s2);
  return coda::launch_status();
}

int coda_bn_relu_bwd_reduce_pooled(long long groups, int group, int c, const float *y, const float *dpooled,
                                   const unsigned char *argmax, const float *mean, const float *invstd,
                                   const float *gamma, const float *beta, float *s1, float *s2, float *scratch,
                                   float *dprime, void *stream) {
  if (groups <= 0 || group < 1 || group > 256 || !channels_ok(c) || !y || !dpooled || !argmax || !mean || !invstd ||
      !gamma || !beta || !s1 || !s2 || !scratch)
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(groups, c);
  bn_relu_bwd_reduce_pooled_kernel<<<grid, THREADS, 0, s>>>(groups, group, c, y, dpooled, argmax, mean, invstd, gamma,
                                                           beta, scratch, dprime);
  sums_finalize_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, c, scratch, s1, s2);
  return coda::launch_status();
}

int coda_bn_relu_bwd_pack(long long rows, int c, int nsplit, const float *y, const float *dz,
                          const float *dpooled, const unsigned char *argmax, int group, const float *mean,
                          const float *invstd, const float *gamma, const float *beta, const float *s1,
                          const float *s2, void *planes, void *stream) {
  if (rows < 0 || !channels_ok(c) || c % 64 != 0 || nsplit < 1 || nsplit > 3) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!y || !mean || !invstd || !gamma || !beta || !s1 || !s2 || !planes) return CODA_EINVAL;
  const bool pooled = dz == nullptr;
  if (pooled && (!dpooled || !argmax || group < 1 || group > 256 || rows % group != 0)) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  __nv_bfloat16 *p = (__nv_bfloat16 *)planes;
#define CODA_LAUNCH(NS, P) \
  bn_relu_bwd_pack_kernel<NS, P><<<grid, THREADS, 0, s>>>(rows, c, y, dz, dpooled, argmax, group, mean, invstd, gamma, \
                                                          beta, s1, s2, p)
  if (pooled) {
    if (nsplit == 1) CODA_LAUNCH(1, true); else if (nsplit == 2) CODA_LAUNCH(2, true); else CODA_LAUNCH(3, true);
  } else {
    if (nsplit == 1) CODA_LAUNCH(1, false); else if (nsplit == 2) CODA_LAUNCH(2, false); else CODA_LAUNCH(3, false);
  }
#undef CODA_LAUNCH
  return coda::launch_status();
}

int coda_bn_relu_bwd_small_k(long long rows, int cin, int cout, const float *y, const float *dz, const float *mean,
                             const float *invstd, const float *gamma, const float *beta, const float *s1,
                             const float *s2, const float *x, float *dw, float *scratch, void *stream) {
  if (rows <= 0 || cin < 1 || cin > 8 || !channels_ok(cout)) return CODA_EINVAL;
  if (!y || !dz || !mean || !invstd || !gamma || !beta || !s1 || !s2 || !x || !dw || !scratch) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, cout);
#define CODA_CASE(K)                                                                                              \
  case K:                                                                                                         \
    bn_relu_bwd_small_k_kernel<K><<<grid, THREADS, 0, s>>>(rows, cout, y, dz, mean, invstd, gamma, beta, s1, s2, x, \
                                                           scratch);                                             \
    break;
  switch (cin) { CODA_CASE(1) CODA_CASE(2) CODA_CASE(3) CODA_CASE(4) CODA_CASE(5) CODA_CASE(6) CODA_CASE(7) CODA_CASE(8) }
#undef CODA_CASE
  dw_finalize_kernel<<<(cin * cout + 127) / 128, 128, 0, s>>>((int)grid, cin * cout, scratch, dw);
  return coda::launch_status();
}

}  // extern "C"
