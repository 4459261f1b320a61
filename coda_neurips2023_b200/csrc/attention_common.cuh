// Shared pieces of the wgmma attention kernels (forward: attention_sm90.cu, backward:
// attention_bwd_sm90.cu): tile sizes, split-product tables, bf16 plane splitting, dropout hash.
#pragma once
#include <math.h>

#include "sm90_primitives.cuh"

namespace coda {
namespace attn {

constexpr int QT = 128;   // queries per CTA
constexpr int KT = 64;    // keys per tile (one 128-byte swizzle span of bf16)
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__host__ __device__ constexpr int a_nprod(int ns) { return ns == 1 ? 1 : (ns == 2 ? 3 : 6); }
__host__ __device__ constexpr int a_pa(int ns, int p) {
  return ns == 1 ? 0 : ns == 2 ? (p == 0 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 2 : p == 2 ? 0 : p == 3 ? 1 : 0);
}
__host__ __device__ constexpr int a_pb(int ns, int p) {
  return ns == 1 ? 0 : ns == 2 ? (p == 1 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 0 : p == 2 ? 2 : p == 3 ? 0 : p == 4 ? 1 : 0);
}

// ------------------------------------------------------------------ operand packing
// src (L, B, H*HD) fp32 sequence-first.  mode 0: planes [ns][B*H][L][HD]   (q, k; K-major rows)
//                                        mode 1: planes [ns][B*H][HD][Lpad] (v^T; keys contiguous)
template <int NSPLIT>
__device__ __forceinline__ void split3(float x, __nv_bfloat16 *dst, size_t plane_stride) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  dst[0] = h;
  if (NSPLIT >= 2) {
    const float r1 = x - __bfloat162float(h);
    const __nv_bfloat16 m = __float2bfloat16_rn(r1);
    dst[plane_stride] = m;
    if (NSPLIT >= 3) dst[2 * plane_stride] = __float2bfloat16_rn(r1 - __bfloat162float(m));
  }
}

// Several (L, B, H*hd) tensors (fp32 or fp16, row stride `ld` elements: slices of a fused qkv projection are
// read in place) -> row planes [NS][B*H][L][hd] in ONE launch: blockIdx.y selects the tensor, a thread converts
// four consecutive head-dim elements (one 16- or 8-byte load, one 8-byte store per plane).
struct PackJob {
  const void *src;
  __nv_bfloat16 *planes;
  int L;
  float scale;
  long long ld;     // elements between consecutive (l, b) rows of src
};
struct PackJobs {
  PackJob job[4];
};
template <int NSPLIT, bool HALF_IN>
__global__ void __launch_bounds__(256)
pack_rows_multi_kernel(const __grid_constant__ PackJobs jobs, int B, int H, int hd) {
  const PackJob jb = jobs.job[blockIdx.y];
  const long long total4 = (long long)jb.L * B * H * hd / 4;
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= total4) return;
  const int hd4 = hd >> 2;
  const int d = (int)(i4 % hd4) * 4;
  long long t = i4 / hd4;
  const int h = (int)(t % H); t /= H;     // t = l * B + b
  const int b = (int)(t % B);
  const int l = (int)(t / B);
  const long long off = t * jb.ld + (long long)h * hd + d;
  float r[4];
  if (HALF_IN) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(static_cast<const __half *>(jb.src) + off));
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
    r[0] = lo.x * jb.scale; r[1] = lo.y * jb.scale; r[2] = hi.x * jb.scale; r[3] = hi.y * jb.scale;
  } else {
    const float4 v = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(jb.src) + off));
    r[0] = v.x * jb.scale; r[1] = v.y * jb.scale; r[2] = v.z * jb.scale; r[3] = v.w * jb.scale;
  }
  __nv_bfloat16 *dst = jb.planes + (((size_t)(b * H + h)) * jb.L + l) * hd + d;
  const size_t plane_stride = (size_t)total4 * 4;
#pragma unroll
  for (int p = 0; p < NSPLIT; ++p) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(r[0], r[1]), hi = __floats2bfloat162_rn(r[2], r[3]);
    uint2 w;
    w.x = *reinterpret_cast<const uint32_t *>(&lo);
    w.y = *reinterpret_cast<const uint32_t *>(&hi);
    *reinterpret_cast<uint2 *>(dst + (size_t)p * plane_stride) = w;
    if (p + 1 < NSPLIT) {
      r[0] -= __uint_as_float(w.x << 16); r[1] -= __uint_as_float(w.x & 0xFFFF0000u);
      r[2] -= __uint_as_float(w.y << 16); r[3] -= __uint_as_float(w.y & 0xFFFF0000u);
    }
  }
}

// ------------------------------------------------------------------ dropout mask (counter hash)
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12; h *= 0x297A2D39u; h ^= h >> 15;
  return h;
}
// keep-decision of element (bh, q, k).  One strong hash per (row, 64-key tile) seeds a 32-bit LCG that is
// stepped along the keys (x_c = A^(c+1) s + C (A^c + ... + 1), available in closed form for any c), and an
// element is kept when x_c >= p * 2^32.  The forward kernel walks the sequence with one IMAD per element;
// attention_launch.py (dropout_keep) restates the same formula for the reference twin.
constexpr uint32_t LCG_A = 747796405u, LCG_C = 2891336453u;
struct LcgJump {
  uint32_t a[KT], c[KT];
};
__host__ __device__ constexpr LcgJump make_lcg_jump() {
  LcgJump t{};
  uint32_t a = LCG_A, c = LCG_C;
  for (int i = 0; i < KT; ++i) {
    t.a[i] = a;
    t.c[i] = c;
    c = c * LCG_A + LCG_C;
    a = a * LCG_A;
  }
  return t;
}
static __constant__ LcgJump kLcgJump = make_lcg_jump();

__host__ __device__ __forceinline__ uint32_t drop_thresh32(float drop_p) {
  return (uint32_t)((double)drop_p * 4294967296.0);
}
__device__ __forceinline__ uint32_t drop_tile_seed(uint32_t seed, uint32_t bh, uint32_t q, uint32_t tile) {
  return mix32(seed + bh * 0x9E3779B1u + q * 0x85EBCA77u + tile * 0xC2B2AE3Du);
}
__device__ __forceinline__ bool drop_keep(uint32_t seed, uint32_t bh, uint32_t q, uint32_t k, uint32_t thresh32) {
  const uint32_t s = drop_tile_seed(seed, bh, q, k / KT);
  return s * kLcgJump.a[k % KT] + kLcgJump.c[k % KT] >= thresh32;
}


}  // namespace attn
}  // namespace coda
