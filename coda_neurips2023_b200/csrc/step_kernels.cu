// Step-glue kernels for H100 (sm_90a): residual + dropout, BatchNorm(+ReLU+dropout) on channels-last rows
// with an fp32 result (the GenericMLP blocks), global-norm clip + AdamW on the flat parameter buffer.
// All of them are pure streaming kernels over L2-resident or HBM-resident fp32 tensors: float4 per thread,
// grid sized in multiples of the SM count, per-channel parameters in registers.  C-ABI in include/coda_step.h.
#include <math.h>
#include <stdint.h>

#include "../../include/coda_sa_mlp.h"
#include "../../include/coda_step.h"
#include "coda_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int NUM_SMS = 132;   // H100 SXM

// ------------------------------------------------------------------ counter-based dropout mask
// One 32-bit draw per element: lowbias32-style avalanche of (seed + index * odd).  Fwd and bwd call this with
// the same (seed, salt, index) and therefore see the same mask.
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du;
  x ^= x >> 15; x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}
struct Drop {
  uint32_t key, thresh;
  float scale;
  bool on;
  __device__ __forceinline__ Drop(float p, unsigned salt, const unsigned *seed) {
    on = p > 0.f;
    key = on ? mix32((seed ? __ldg(seed) : 0u) + salt * 0x9E3779B1u) : 0u;
    thresh = (uint32_t)fminf(p * 4294967296.0f, 4294967040.0f);
    scale = on ? 1.0f / (1.0f - p) : 1.0f;
  }
  // multiplier of element `i`
  __device__ __forceinline__ float operator()(unsigned long long i) const {
    if (!on) return 1.0f;
    const uint32_t h = mix32(key ^ mix32((uint32_t)i * 0x85EBCA77u + (uint32_t)(i >> 32) * 0xC2B2AE3Du + 0x27D4EB2Fu));
    return h >= thresh ? scale : 0.0f;
  }
};

__host__ inline unsigned stream_grid(long long work_items) {
  const long long need = (work_items + THREADS - 1) / THREADS;
  const long long cap = NUM_SMS * 8;
  return (unsigned)(need < cap ? (need > 0 ? need : 1) : cap);
}

__global__ void __launch_bounds__(THREADS)
dropout_add_kernel(long long n, const float *__restrict__ x, const float *__restrict__ resid, float p, unsigned salt,
                   const unsigned *__restrict__ seed, float *__restrict__ out) {
  const Drop drop(p, salt, seed);
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    float4 v = __ldg(reinterpret_cast<const float4 *>(x) + i);
    v.x *= drop(4 * i); v.y *= drop(4 * i + 1); v.z *= drop(4 * i + 2); v.w *= drop(4 * i + 3);
    if (resid) {
      const float4 r = __ldg(reinterpret_cast<const float4 *>(resid) + i);
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    reinterpret_cast<float4 *>(out)[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    out[i] = x[i] * drop(i) + (resid ? resid[i] : 0.f);
  }
}

// ------------------------------------------------------------------ BatchNorm (+ReLU, +dropout) on rows, fp32 out
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
__host__ __device__ inline bool channels_ok(int c) { return c >= 4 && c <= 1024 && c % 4 == 0 && THREADS % (c / 4) == 0; }
constexpr int MAX_BLOCKS = NUM_SMS * 4;   // must match coda_bn_rows_scratch_floats (sa_mlp_kernels.cu)
__host__ inline unsigned grid_for(long long rows, int c) {
  const long long per_iter = THREADS / (c / 4);
  const long long need = (rows + per_iter - 1) / per_iter;
  return (unsigned)(need < MAX_BLOCKS ? (need > 0 ? need : 1) : MAX_BLOCKS);
}

// the gradient that reaches the BatchNorm output: dout through the dropout and ReLU masks
__device__ __forceinline__ float4 masked_grad(float4 d, const float4 z, int relu, const Drop &drop, unsigned long long e0) {
  d.x *= drop(e0); d.y *= drop(e0 + 1); d.z *= drop(e0 + 2); d.w *= drop(e0 + 3);
  if (relu) {
    d.x = z.x > 0.f ? d.x : 0.f; d.y = z.y > 0.f ? d.y : 0.f; d.z = z.z > 0.f ? d.z : 0.f; d.w = z.w > 0.f ? d.w : 0.f;
  }
  return d;
}

__global__ void __launch_bounds__(THREADS)
bn_act_fwd_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ mean,
                  const float *__restrict__ invstd, const float *__restrict__ gamma, const float *__restrict__ beta,
                  int relu, float p, unsigned salt, const unsigned *__restrict__ seed, float *__restrict__ out) {
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const Drop drop(p, salt, seed);
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    float4 z = bn4(xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a), a);
    if (relu) { z.x = fmaxf(z.x, 0.f); z.y = fmaxf(z.y, 0.f); z.z = fmaxf(z.z, 0.f); z.w = fmaxf(z.w, 0.f); }
    const unsigned long long e0 = (unsigned long long)r * c + c4 * 4;
    z.x *= drop(e0); z.y *= drop(e0 + 1); z.z *= drop(e0 + 2); z.w *= drop(e0 + 3);
    reinterpret_cast<float4 *>(out + r * c)[c4] = z;
  }
}

__global__ void __launch_bounds__(THREADS)
bn_act_bwd_reduce_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ dout,
                         const float *__restrict__ mean, const float *__restrict__ invstd,
                         const float *__restrict__ gamma, const float *__restrict__ beta, int relu, float p,
                         unsigned salt, const unsigned *__restrict__ seed, float *__restrict__ partial) {
  __shared__ float4 red[THREADS];
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const Drop drop(p, salt, seed);
  float4 acc[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 xh = xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a);
    const float4 d = masked_grad(__ldg(reinterpret_cast<const float4 *>(dout + r * c) + c4), bn4(xh, a), relu, drop,
                                 (unsigned long long)r * c + c4 * 4);
    acc[0].x += d.x; acc[0].y += d.y; acc[0].z += d.z; acc[0].w += d.w;
    acc[1].x = fmaf(d.x, xh.x, acc[1].x); acc[1].y = fmaf(d.y, xh.y, acc[1].y);
    acc[1].z = fmaf(d.z, xh.z, acc[1].z); acc[1].w = fmaf(d.w, xh.w, acc[1].w);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    __syncthreads();
    red[threadIdx.x] = acc[i];
    __syncthreads();
    if (slot == 0) {
      float4 t = acc[i];
      for (int s = 1; s < nslots; ++s) {
        const float4 o = red[s * cq + c4];
        t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w;
      }
      reinterpret_cast<float4 *>(partial + (size_t)blockIdx.x * 2 * c + (size_t)i * c)[c4] = t;
    }
  }
}
// one warp per channel: lanes stride over the block partials (fp64), then a shuffle tree
__global__ void __launch_bounds__(256)
sums_finalize_kernel(int nblocks, int c, const float *__restrict__ partial, float *__restrict__ s1,
                     float *__restrict__ s2) {
  const int ch = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (ch >= c) return;
  double a = 0.0, b = 0.0;
  for (int k = lane; k < nblocks; k += 32) {
    a += (double)partial[(size_t)k * 2 * c + ch];
    b += (double)partial[(size_t)k * 2 * c + c + ch];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    s1[ch] = (float)a;
    s2[ch] = (float)b;
  }
}

__global__ void __launch_bounds__(THREADS)
bn_act_bwd_kernel(long long rows, int c, const float *__restrict__ y, const float *__restrict__ dout,
                  const float *__restrict__ mean, const float *__restrict__ invstd, const float *__restrict__ gamma,
                  const float *__restrict__ beta, int relu, float p, unsigned salt, const unsigned *__restrict__ seed,
                  const float *__restrict__ s1, const float *__restrict__ s2, float *__restrict__ dy) {
  const int cq = c >> 2, c4 = threadIdx.x % cq, slot = threadIdx.x / cq, nslots = THREADS / cq;
  const Affine4 a = load_affine(mean, invstd, gamma, beta, c4);
  const Drop drop(p, salt, seed);
  const float inv_n = 1.0f / (float)rows;
  const float4 t1 = __ldg(reinterpret_cast<const float4 *>(s1) + c4), t2 = __ldg(reinterpret_cast<const float4 *>(s2) + c4);
  const float4 k = make_float4(a.gamma.x * a.invstd.x, a.gamma.y * a.invstd.y, a.gamma.z * a.invstd.z, a.gamma.w * a.invstd.w);
  const float4 m1 = make_float4(t1.x * inv_n, t1.y * inv_n, t1.z * inv_n, t1.w * inv_n);
  const float4 m2 = make_float4(t2.x * inv_n, t2.y * inv_n, t2.z * inv_n, t2.w * inv_n);
  for (long long r = (long long)blockIdx.x * nslots + slot; r < rows; r += (long long)gridDim.x * nslots) {
    const float4 xh = xhat4(__ldg(reinterpret_cast<const float4 *>(y + r * c) + c4), a);
    const float4 d = masked_grad(__ldg(reinterpret_cast<const float4 *>(dout + r * c) + c4), bn4(xh, a), relu, drop,
                                 (unsigned long long)r * c + c4 * 4);
    reinterpret_cast<float4 *>(dy + r * c)[c4] =
        make_float4(k.x * (d.x - m1.x - xh.x * m2.x), k.y * (d.y - m1.y - xh.y * m2.y),
                    k.z * (d.z - m1.z - xh.z * m2.z), k.w * (d.w - m1.w - xh.w * m2.w));
  }
}

// ------------------------------------------------------------------ global-norm clip + AdamW
constexpr int NORM_BLOCKS = NUM_SMS * 4;

__global__ void __launch_bounds__(THREADS)
sumsq_partial_kernel(long long n, const float *__restrict__ g, float *__restrict__ partial) {
  __shared__ float red[THREADS / 32];
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    const float4 v = __ldg(reinterpret_cast<const float4 *>(g) + i);
    a0 = fmaf(v.x, v.x, a0); a1 = fmaf(v.y, v.y, a1); a2 = fmaf(v.z, v.z, a2); a3 = fmaf(v.w, v.w, a3);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = g[(n4 << 2) + threadIdx.x];
    a0 = fmaf(v, v, a0);
  }
  float a = (a0 + a1) + (a2 + a3);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) t += red[w];
    partial[blockIdx.x] = t;
  }
}
// one warp: fp64 sum of the block partials -> norm, clip coefficient, step counter, bias corrections
__global__ void norm_finalize_kernel(int nblocks, const float *__restrict__ partial, float grad_scale, float max_norm,
                                     float beta1, float beta2, float *__restrict__ state) {
  double a = 0.0;
  for (int k = threadIdx.x; k < nblocks; k += 32) a += (double)partial[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (threadIdx.x == 0) {
    const double norm = sqrt(a) * fabs((double)grad_scale);
    const float step = state[0] + 1.0f;
    state[0] = step;
    state[1] = (float)norm;
    // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
    state[2] = max_norm > 0.f ? fminf((float)((double)max_norm / (norm + 1e-6)), 1.0f) : 1.0f;
    state[3] = (float)(1.0 - pow((double)beta1, (double)step));
    state[4] = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  }
}

__global__ void __launch_bounds__(THREADS)
adamw_kernel(int nchunks, const coda_opt_chunk *__restrict__ chunks, float *__restrict__ param,
             const float *__restrict__ grad, float *__restrict__ exp_avg, float *__restrict__ exp_avg_sq,
             const float *__restrict__ lr_dev, float grad_scale, float beta1, float beta2, float eps,
             const float *__restrict__ state) {
  const float lr = __ldg(lr_dev);
  const float gs = grad_scale * __ldg(state + 2);
  const float step_size = lr / __ldg(state + 3);
  const float inv_sqrt_bc2 = 1.0f / __ldg(state + 4);
  for (int ci = blockIdx.x; ci < nchunks; ci += gridDim.x) {
    const coda_opt_chunk ch = chunks[ci];
    const float decay = 1.0f - lr * ch.weight_decay;
    float *p = param + ch.offset, *m = exp_avg + ch.offset, *v = exp_avg_sq + ch.offset;
    const float *g = grad + ch.offset;
    // chunk offsets are multiples of 4 except at tensor boundaries: scalar head / tail around an aligned body
    const int head = (int)((4 - (ch.offset & 3)) & 3) < ch.len ? (int)((4 - (ch.offset & 3)) & 3) : ch.len;
    auto upd = [&](float &pp, float &mm, float &vv, float gg) {
      gg *= gs;
      pp *= decay;
      mm += (gg - mm) * (1.0f - beta1);
      vv = beta2 * vv + (1.0f - beta2) * gg * gg;
      pp -= step_size * mm / (sqrtf(vv) * inv_sqrt_bc2 + eps);
    };
    if (threadIdx.x < head) upd(p[threadIdx.x], m[threadIdx.x], v[threadIdx.x], g[threadIdx.x]);
    const int body4 = (ch.len - head) >> 2;
    for (int i = threadIdx.x; i < body4; i += THREADS) {
      float4 pv = reinterpret_cast<float4 *>(p + head)[i], mv = reinterpret_cast<float4 *>(m + head)[i];
      float4 vv = reinterpret_cast<float4 *>(v + head)[i];
      const float4 gv = __ldg(reinterpret_cast<const float4 *>(g + head) + i);
      upd(pv.x, mv.x, vv.x, gv.x); upd(pv.y, mv.y, vv.y, gv.y); upd(pv.z, mv.z, vv.z, gv.z); upd(pv.w, mv.w, vv.w, gv.w);
      reinterpret_cast<float4 *>(p + head)[i] = pv;
      reinterpret_cast<float4 *>(m + head)[i] = mv;
      reinterpret_cast<float4 *>(v + head)[i] = vv;
    }
    const int tail0 = head + (body4 << 2);
    if (threadIdx.x < ch.len - tail0) {
      const int i = tail0 + threadIdx.x;
      upd(p[i], m[i], v[i], g[i]);
    }
  }
}

// ------------------------------------------------------------------ n-ary gradient sum
// out = src[0] + src[1] + ... + src[count - 1]: the fan-in of a tensor that several branches consumed (the six
// prediction heads on the decoder output, the sixteen uses of the query embedding) as ONE pass that reads each
// contribution once, instead of count - 1 `a + b` kernels that re-read and re-write the running sum.
constexpr int SUM_MAX = 16;
struct SumSrcs {
  const float *p[SUM_MAX];
};
__global__ void __launch_bounds__(THREADS)
sum_n_kernel(long long n, int count, const SumSrcs srcs, float *__restrict__ out) {
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    float4 a = __ldg(reinterpret_cast<const float4 *>(srcs.p[0]) + i);
    for (int j = 1; j < count; ++j) {
      const float4 t = __ldg(reinterpret_cast<const float4 *>(srcs.p[j]) + i);
      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
    }
    reinterpret_cast<float4 *>(out)[i] = a;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    float a = srcs.p[0][i];
    for (int j = 1; j < count; ++j) a += srcs.p[j][i];
    out[i] = a;
  }
}

// ------------------------------------------------------------------ masked L1 (cross-modal alignment loss)
// out[l] = sum_{r, d} | pred[l][r][d] * w[r] - target[r][d] * w[r] |   (criterion.py:924-943: the products are formed
// separately, as the reference does, so the value rounds the same way).  Two-stage deterministic sum.
constexpr int L1_BLOCKS = 128;   // per layer
__global__ void __launch_bounds__(THREADS)
masked_l1_fwd_kernel(long long rows, int d, const float *__restrict__ pred, const float *__restrict__ target,
                     const float *__restrict__ w, float *__restrict__ partial) {
  const int layer = blockIdx.y;
  const int d4 = d >> 2;
  const long long n4 = rows * d4;
  const float4 *p4 = reinterpret_cast<const float4 *>(pred) + (long long)layer * n4;
  const float4 *t4 = reinterpret_cast<const float4 *>(target);
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    const float wr = __ldg(w + i / d4);
    const float4 a = __ldg(p4 + i), b = __ldg(t4 + i);
    acc += (fabsf(a.x * wr - b.x * wr) + fabsf(a.y * wr - b.y * wr)) +
           (fabsf(a.z * wr - b.z * wr) + fabsf(a.w * wr - b.w * wr));
  }
  __shared__ float red[THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < THREADS / 32; ++k) t += red[k];
    partial[(long long)layer * gridDim.x + blockIdx.x] = t;
  }
}
__global__ void masked_l1_finalize_kernel(int nblocks, const float *__restrict__ partial, float *__restrict__ out) {
  double a = 0.0;
  for (int k = threadIdx.x; k < nblocks; k += 32) a += (double)partial[(long long)blockIdx.x * nblocks + k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (threadIdx.x == 0) out[blockIdx.x] = (float)a;
}
// dpred[l][r][d] = g[l] * sgn(pred * w - target * w) * w[r]
__global__ void __launch_bounds__(THREADS)
masked_l1_bwd_kernel(long long rows, int d, const float *__restrict__ pred, const float *__restrict__ target,
                     const float *__restrict__ w, const float *__restrict__ g, float *__restrict__ dpred) {
  const int layer = blockIdx.y;
  const int d4 = d >> 2;
  const long long n4 = rows * d4;
  const float4 *p4 = reinterpret_cast<const float4 *>(pred) + (long long)layer * n4;
  const float4 *t4 = reinterpret_cast<const float4 *>(target);
  float4 *o4 = reinterpret_cast<float4 *>(dpred) + (long long)layer * n4;
  const float gl = __ldg(g + layer);
  auto sgn = [](float v) { return (float)((v > 0.f) - (v < 0.f)); };
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    const float wr = __ldg(w + i / d4);
    const float4 a = __ldg(p4 + i), b = __ldg(t4 + i);
    const float gw = gl * wr;
    float4 o;
    o.x = sgn(a.x * wr - b.x * wr) * gw;
    o.y = sgn(a.y * wr - b.y * wr) * gw;
    o.z = sgn(a.z * wr - b.z * wr) * gw;
    o.w = sgn(a.w * wr - b.w * wr) * gw;
    o4[i] = o;
  }
}

}  // namespace

extern "C" {

int coda_dropout_add_fwd(long long n, const float *x, const float *resid, float p, unsigned salt, const unsigned *seed,
                         float *out, void *stream) {
  if (n < 0 || p < 0.f || p >= 1.f) return CODA_EINVAL;
  if (n == 0) return CODA_OK;
  if (!x || !out || (((uintptr_t)x | (uintptr_t)out | (uintptr_t)resid) & 15)) return CODA_EINVAL;
  dropout_add_kernel<<<stream_grid(n / 4 + 1), THREADS, 0, (cudaStream_t)stream>>>(n, x, resid, p, salt, seed, out);
  return coda::launch_status();
}

int coda_dropout_bwd(long long n, const float *dout, float p, unsigned salt, const unsigned *seed, float *dx,
                     void *stream) {
  return coda_dropout_add_fwd(n, dout, nullptr, p, salt, seed, dx, stream);
}

int coda_bn_act_rows_fwd(long long rows, int c, const float *y, const float *mean, const float *invstd,
                         const float *gamma, const float *beta, int relu, float p, unsigned salt, const unsigned *seed,
                         float *out, void *stream) {
  if (rows < 0 || !channels_ok(c) || p < 0.f || p >= 1.f) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!y || !mean || !invstd || !gamma || !beta || !out) return CODA_EINVAL;
  bn_act_fwd_kernel<<<grid_for(rows, c), THREADS, 0, (cudaStream_t)stream>>>(rows, c, y, mean, invstd, gamma, beta, relu,
                                                                            p, salt, seed, out);
  return coda::launch_status();
}

int coda_bn_act_rows_bwd_reduce(long long rows, int c, const float *y, const float *dout, const float *mean,
                                const float *invstd, const float *gamma, const float *beta, int relu, float p,
                                unsigned salt, const unsigned *seed, float *s1, float *s2, float *scratch,
                                void *stream) {
  if (rows <= 0 || !channels_ok(c) || p < 0.f || p >= 1.f) return CODA_EINVAL;
  if (!y || !dout || !mean || !invstd || !gamma || !beta || !s1 || !s2 || !scratch) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned grid = grid_for(rows, c);
  bn_act_bwd_reduce_kernel<<<grid, THREADS, 0, s>>>(rows, c, y, dout, mean, invstd, gamma, beta, relu, p, salt, seed,
                                                    scratch);
  sums_finalize_kernel<<<(c + 7) / 8, 256, 0, s>>>((int)grid, c, scratch, s1, s2);
  return coda::launch_status();
}

int coda_bn_act_rows_bwd(long long rows, int c, const float *y, const float *dout, const float *mean,
                         const float *invstd, const float *gamma, const float *beta, int relu, float p, unsigned salt,
                         const unsigned *seed, const float *s1, const float *s2, float *dy, void *stream) {
  if (rows < 0 || !channels_ok(c) || p < 0.f || p >= 1.f) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!y || !dout || !mean || !invstd || !gamma || !beta || !s1 || !s2 || !dy) return CODA_EINVAL;
  bn_act_bwd_kernel<<<grid_for(rows, c), THREADS, 0, (cudaStream_t)stream>>>(rows, c, y, dout, mean, invstd, gamma, beta,
                                                                            relu, p, salt, seed, s1, s2, dy);
  return coda::launch_status();
}

long long coda_grad_norm_scratch_floats(void) { return NORM_BLOCKS; }

int coda_grad_norm(long long n, const float *grad, float grad_scale, float max_norm, float beta1, float beta2,
                   float *scratch, float *state, void *stream) {
  if (n <= 0 || !grad || !scratch || !state || ((uintptr_t)grad & 15)) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const long long need = (n / 4 + THREADS - 1) / THREADS;
  const int grid = (int)(need < NORM_BLOCKS ? (need > 0 ? need : 1) : NORM_BLOCKS);
  sumsq_partial_kernel<<<grid, THREADS, 0, s>>>(n, grad, scratch);
  norm_finalize_kernel<<<1, 32, 0, s>>>(grid, scratch, grad_scale, max_norm, beta1, beta2, state);
  return coda::launch_status();
}

int coda_adamw_update(int nchunks, const coda_opt_chunk *chunks, float *param, const float *grad, float *exp_avg,
                      float *exp_avg_sq, const float *lr_dev, float grad_scale, float beta1, float beta2, float eps,
                      const float *state, void *stream) {
  if (nchunks < 0) return CODA_EINVAL;
  if (nchunks == 0) return CODA_OK;
  if (!chunks || !param || !grad || !exp_avg || !exp_avg_sq || !lr_dev || !state) return CODA_EINVAL;
  if (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) return CODA_EINVAL;
  const int grid = nchunks < NUM_SMS * 8 ? nchunks : NUM_SMS * 8;
  adamw_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(nchunks, chunks, param, grad, exp_avg, exp_avg_sq, lr_dev,
                                                          grad_scale, beta1, beta2, eps, state);
  return coda::launch_status();
}

int coda_sum_n(long long n, int count, const float *const *srcs, float *out, void *stream) {
  if (n < 0 || count < 1 || count > SUM_MAX || !srcs) return CODA_EINVAL;
  if (n == 0) return CODA_OK;
  if (!out || ((uintptr_t)out & 15)) return CODA_EINVAL;
  SumSrcs a;
  for (int j = 0; j < SUM_MAX; ++j) {
    a.p[j] = srcs[j < count ? j : 0];
    if (!a.p[j] || ((uintptr_t)a.p[j] & 15)) return CODA_EINVAL;
  }
  sum_n_kernel<<<stream_grid(n / 4 + 1), THREADS, 0, (cudaStream_t)stream>>>(n, count, a, out);
  return coda::launch_status();
}

long long coda_masked_l1_scratch_floats(int layers) { return (long long)(layers > 0 ? layers : 0) * L1_BLOCKS; }

int coda_masked_l1_fwd(int layers, long long rows, int d, const float *pred, const float *target, const float *w,
                       float *out, float *scratch, void *stream) {
  if (layers < 0 || rows < 0 || d <= 0 || (d & 3)) return CODA_EINVAL;
  if (layers == 0) return CODA_OK;
  // with no rows the operands are empty (and may be NULL): every out[l] is 0
  if ((rows > 0 && (!pred || !target || !w)) || !out || !scratch || (((uintptr_t)pred | (uintptr_t)target) & 15))
    return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  masked_l1_fwd_kernel<<<dim3(L1_BLOCKS, layers), THREADS, 0, s>>>(rows, d, pred, target, w, scratch);
  int st = coda::launch_status();
  if (st != CODA_OK) return st;
  masked_l1_finalize_kernel<<<layers, 32, 0, s>>>(L1_BLOCKS, scratch, out);
  return coda::launch_status();
}

int coda_masked_l1_bwd(int layers, long long rows, int d, const float *pred, const float *target, const float *w,
                       const float *g, float *dpred, void *stream) {
  if (layers < 0 || rows < 0 || d <= 0 || (d & 3)) return CODA_EINVAL;
  if (layers == 0 || rows == 0) return CODA_OK;
  if (!pred || !target || !w || !g || !dpred || (((uintptr_t)pred | (uintptr_t)target | (uintptr_t)dpred) & 15))
    return CODA_EINVAL;
  masked_l1_bwd_kernel<<<dim3(L1_BLOCKS, layers), THREADS, 0, (cudaStream_t)stream>>>(rows, d, pred, target, w, g,
                                                                                      dpred);
  return coda::launch_status();
}

}  // extern "C"
