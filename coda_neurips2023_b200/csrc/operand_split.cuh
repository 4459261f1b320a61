// The split-bf16 operand format of the tensor-core kernels, defined once.
//
// An fp32 value x is carried as NP bf16 planes, x = p0 + p1 (+ p2): plane p is the bf16 rounding (round to nearest
// even) of what the planes before it left over.  Two planes carry ~16 mantissa bits, three the full 24.  A product of
// two operands split into the same number of planes is the sum of the plane products listed by n_products / prod_a /
// prod_b, small terms first.  Pack kernels and in-register prologues write planes only through the functions below.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace coda {

// two floats -> one register of two 16-bit values (low half = first), bf16 or IEEE half
template <bool F16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (F16) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
  } else {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
  }
}

// the next plane of a pair of remainders: their bf16 roundings, packed; r0, r1 keep what the plane leaves over
__device__ __forceinline__ uint32_t next_plane(float &r0, float &r1) {
  const uint32_t bits = pack2<false>(r0, r1);
  r0 -= __uint_as_float(bits << 16);
  r1 -= __uint_as_float(bits & 0xFFFF0000u);
  return bits;
}

// a pair of values -> NP bf16 planes (plane p = bf16 rounding of what the previous planes left over)
template <int NP>
__device__ __forceinline__ void split_pair(float r0, float r1, uint32_t (&w)[NP]) {
#pragma unroll
  for (int p = 0; p < NP; ++p) w[p] = next_plane(r0, r1);
}

// four consecutive values -> NP planes, one 8-byte store per plane (dst 8-byte aligned; plane_stride in elements)
template <int NP>
__device__ __forceinline__ void split_store4(float4 v, __nv_bfloat16 *dst, size_t plane_stride) {
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const uint32_t lo = next_plane(v.x, v.y), hi = next_plane(v.z, v.w);
    *reinterpret_cast<uint2 *>(dst + (size_t)p * plane_stride) = make_uint2(lo, hi);
  }
}

// one value -> NP planes, for the pack kernels whose threads own single elements
template <int NP>
__device__ __forceinline__ void split_store(float x, __nv_bfloat16 *dst, size_t plane_stride) {
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    dst[p * plane_stride] = h;
    if (p + 1 < NP) x -= __bfloat162float(h);
  }
}

// which (A plane, B plane) pairs are multiplied for NP planes per operand; small cross terms first
__host__ __device__ constexpr int n_products(int np) { return np == 1 ? 1 : (np == 2 ? 3 : 6); }
__host__ __device__ constexpr int prod_a(int np, int p) {
  return np == 1 ? 0 : np == 2 ? (p == 0 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 2 : p == 2 ? 0 : p == 3 ? 1 : 0);
}
__host__ __device__ constexpr int prod_b(int np, int p) {
  return np == 1 ? 0 : np == 2 ? (p == 1 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 0 : p == 2 ? 2 : p == 3 ? 0 : p == 4 ? 1 : 0);
}

}  // namespace coda
