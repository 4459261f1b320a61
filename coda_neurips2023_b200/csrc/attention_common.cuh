// Shared pieces of the wgmma attention kernels (forward: attention_sm90.cu, backward:
// attention_bwd_sm90.cu): tile sizes, operand packing, dropout hash.
#pragma once
#include <math.h>

#include "sm90_primitives.cuh"

namespace coda {
namespace attn {

constexpr int QT = 128;   // queries per CTA
constexpr int KT = 64;    // keys per tile (one 128-byte swizzle span of bf16)
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

// ------------------------------------------------------------------ operand packing
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
  float4 r;
  if (HALF_IN) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(static_cast<const __half *>(jb.src) + off));
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
    r = make_float4(lo.x * jb.scale, lo.y * jb.scale, hi.x * jb.scale, hi.y * jb.scale);
  } else {
    const float4 v = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(jb.src) + off));
    r = make_float4(v.x * jb.scale, v.y * jb.scale, v.z * jb.scale, v.w * jb.scale);
  }
  split_store4<NSPLIT>(r, jb.planes + (((size_t)(b * H + h)) * jb.L + l) * hd + d, (size_t)total4 * 4);
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
