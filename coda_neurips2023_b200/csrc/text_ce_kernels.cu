// Row-wise cross-entropy of the stage-2 contrastive loss over a shared text matrix, on logits a GEMM has written
// (C-ABI and formulas in include/coda_step.h, coda_text_ce_fwd / coda_text_ce_bwd).  One warp per row: the row of
// S (C = 1201 floats at the scripts' shape) is read with float4 loads, once for the maximum and once more (from L1)
// for the sum; the embedding row (512 floats) gives the norm.  Every reduction is lane-strided then a shuffle tree,
// so a row's result does not depend on the launch or on the other rows.
#include <math.h>
#include <stdint.h>

#include "../../include/coda_step.h"
#include "coda_common.cuh"

namespace {

constexpr int THREADS = 256;
constexpr int ROWS_PER_BLOCK = THREADS / 32;
constexpr long long IGNORE_INDEX = -100;

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

// z = a * S rounded on its own (no contraction into a later subtraction): forward and backward see the same z
__device__ __forceinline__ float logit(float a, float s) { return __fmul_rn(a, s); }

// ||e_r||: the same order in forward and backward, so both see the same bits
__device__ __forceinline__ float row_norm(const float4 *e4, int d4, int lane) {
  float acc = 0.f;
  for (int k = lane; k < d4; k += 32) {
    const float4 v = __ldg(e4 + k);
    acc += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  return sqrtf(warp_sum(acc));
}

__global__ void __launch_bounds__(THREADS)
text_ce_fwd_kernel(long long rows, int c, int ld, int d, const float *__restrict__ S, const float *__restrict__ e,
                   const long long *__restrict__ label, const float *__restrict__ w, const float *__restrict__ scale,
                   float *__restrict__ loss, float *__restrict__ lse_out, float *__restrict__ inv_out) {
  const long long r = (long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float inv = 1.0f / (row_norm(reinterpret_cast<const float4 *>(e + r * d), d >> 2, lane) + 1e-32f);
  const float a = __ldg(scale) * inv;
  const float4 *s4 = reinterpret_cast<const float4 *>(S + r * ld);
  const int n4 = (c + 3) >> 2;
  float m = -INFINITY;
  for (int k = lane; k < n4; k += 32) {
    const float4 v = __ldg(s4 + k);
    const int col = k << 2;
    m = fmaxf(m, logit(a, v.x));
    if (col + 1 < c) m = fmaxf(m, logit(a, v.y));
    if (col + 2 < c) m = fmaxf(m, logit(a, v.z));
    if (col + 3 < c) m = fmaxf(m, logit(a, v.w));
  }
  m = warp_max(m);
  // sum_c exp(z_c - m) = (number of maxima) + rest: lse = m + log1p(rest + maxima - 1) keeps the bits that
  // 1 + rest would round away (a nearly one-hot row)
  float rest = 0.f, maxima = 0.f;
  for (int k = lane; k < n4; k += 32) {
    const float4 v = __ldg(s4 + k);
    const int col = k << 2;
    const float z[4] = {logit(a, v.x), logit(a, v.y), logit(a, v.z), logit(a, v.w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (col + j < c) {
        if (z[j] < m) rest += expf(z[j] - m);
        else maxima += 1.f;
      }
    }
  }
  rest = warp_sum(rest);
  maxima = warp_sum(maxima);
  if (lane == 0) {
    const float lse = m + log1pf(rest + (maxima - 1.f));
    const long long y = __ldg(label + r);
    float out;
    if (y == IGNORE_INDEX) out = 0.f;
    else if (y < 0 || y >= c) out = __int_as_float(0x7fc00000);
    else out = __ldg(w + r) * (lse - logit(a, __ldg(S + r * ld + y)));
    loss[r] = out;
    lse_out[r] = lse;
    inv_out[r] = inv;
  }
}

__global__ void __launch_bounds__(THREADS)
text_ce_bwd_kernel(long long rows, int c, int ld, int d, const float *__restrict__ S, const float *__restrict__ e,
                   const long long *__restrict__ label, const float *__restrict__ w, const float *__restrict__ scale,
                   const float *__restrict__ lse_in, const float *__restrict__ inv_in, const float *__restrict__ g,
                   float *__restrict__ dS, float *__restrict__ dnorm) {
  const long long r = (long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const long long y = __ldg(label + r);
  const float inv = __ldg(inv_in + r);
  const float a = __ldg(scale) * inv;
  const float lse = __ldg(lse_in + r);
  // G_rc = gw * (p_rc - [c == y]); an ignored row has gw = 0, an out-of-range label poisons the row with NaN
  float gw = __ldg(g + r) * __ldg(w + r);
  if (y == IGNORE_INDEX) gw = 0.f;
  else if (y < 0 || y >= c) gw = __int_as_float(0x7fc00000);
  const float4 *s4 = reinterpret_cast<const float4 *>(S + r * ld);
  float4 *o4 = reinterpret_cast<float4 *>(dS + r * ld);
  const int ld4 = ld >> 2;
  const float zy = (y >= 0 && y < c) ? logit(a, __ldg(S + r * ld + y)) : 0.f;
  // sum_c G_rc z_rc = gw * sum_c p_rc (z_rc - z_ry): the same value (sum_c (p_rc - [c == y]) = 0) without the
  // cancellation of sum_c p_rc z_rc against z_ry; p_ry - 1 as expm1 for the same reason
  float gz = 0.f;
  for (int k = lane; k < ld4; k += 32) {
    const float4 v = __ldg(s4 + k);
    const int col = k << 2;
    const float z[4] = {logit(a, v.x), logit(a, v.y), logit(a, v.z), logit(a, v.w)};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (col + j < c) {
        const float q = z[j] - lse;
        const float p = expf(q);
        gz += p * (z[j] - zy);
        o[j] = a * (gw * (col + j == y ? expm1f(q) : p));
      } else {
        o[j] = 0.f;
      }
    }
    o4[k] = make_float4(o[0], o[1], o[2], o[3]);
  }
  gz = gw * warp_sum(gz);
  const float4 *e4 = reinterpret_cast<const float4 *>(e + r * d);
  const int d4 = d >> 2;
  const float n = row_norm(e4, d4, lane);
  const float coef = n > 0.f ? -(inv / n) * gz : 0.f;
  float4 *n4 = reinterpret_cast<float4 *>(dnorm + r * d);
  for (int k = lane; k < d4; k += 32) {
    const float4 v = __ldg(e4 + k);
    n4[k] = make_float4(coef * v.x, coef * v.y, coef * v.z, coef * v.w);
  }
}

bool args_ok(long long rows, int c, int ld, int d) {
  return rows >= 0 && c >= 1 && ld >= c && (ld & 3) == 0 && d > 0 && (d & 3) == 0;
}
bool aligned(const void *p) { return ((uintptr_t)p & 15) == 0; }
long long blocks(long long rows) { return (rows + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK; }

}  // namespace

extern "C" {

int coda_text_ce_fwd(long long rows, int c, int ld, int d, const float *S, const float *e, const long long *label,
                     const float *w, const float *scale, float *loss, float *lse, float *inv, void *stream) {
  if (!args_ok(rows, c, ld, d)) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!S || !e || !label || !w || !scale || !loss || !lse || !inv || !aligned(S) || !aligned(e)) return CODA_EINVAL;
  if (blocks(rows) > 0x7fffffffLL) return CODA_ETOOLARGE;
  text_ce_fwd_kernel<<<(unsigned)blocks(rows), THREADS, 0, (cudaStream_t)stream>>>(rows, c, ld, d, S, e, label, w,
                                                                                  scale, loss, lse, inv);
  return coda::launch_status();
}

int coda_text_ce_bwd(long long rows, int c, int ld, int d, const float *S, const float *e, const long long *label,
                     const float *w, const float *scale, const float *lse, const float *inv, const float *g,
                     float *dS, float *dnorm, void *stream) {
  if (!args_ok(rows, c, ld, d)) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!S || !e || !label || !w || !scale || !lse || !inv || !g || !dS || !dnorm || !aligned(S) || !aligned(e) ||
      !aligned(dS) || !aligned(dnorm))
    return CODA_EINVAL;
  if (blocks(rows) > 0x7fffffffLL) return CODA_ETOOLARGE;
  text_ce_bwd_kernel<<<(unsigned)blocks(rows), THREADS, 0, (cudaStream_t)stream>>>(rows, c, ld, d, S, e, label, w,
                                                                                  scale, lse, inv, g, dS, dnorm);
  return coda::launch_status();
}

}  // extern "C"
