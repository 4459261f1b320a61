// The element formulas of the fp32-operand prologues (CODA_A32_* in include/coda_gemm.h), defined once.
//
// The input gradient dX of a layer comes from gemm_a32_sm90.cu and its weight gradient dW from gemm_tn32_sm90.cu; both
// apply the same prologue to the same operand, so both call these functions.  Each is written with a fixed order of
// fmaf / compare / select: results are the same bits in both kernels.
//
// Per column k: s = scale[k], h = shift[k] (BatchNorm folded to an affine, s = gamma * invstd, h = beta - mean * s);
// al = alpha[k], be = beta[k] of the BatchNorm backward (host: coda_bn_bwd_coefs):
//   y = pre-BN activation, d = gradient of relu(bn(y)):
//   dy = s * ([s y + h > 0] d - s1/N - xhat s2/N) = [s y + h > 0] * s * d + al * y + be
//   al = -s * invstd * s2 / N,  be = -s * s1 / N - al * mean
// CODA_A32_PLAIN is the identity and has no function.
#pragma once

namespace coda {
namespace a32 {

// CODA_A32_AFFINE_RELU: BatchNorm (statistics folded into s, h) + ReLU of the previous layer
__device__ __forceinline__ float affine_relu(float x, float s, float h) { return fmaxf(fmaf(x, s, h), 0.f); }

// CODA_A32_BN_BWD: BatchNorm + ReLU backward, dense gradient d
__device__ __forceinline__ float bn_bwd(float y, float d, float s, float h, float al, float be) {
  return (fmaf(y, s, h) > 0.f ? s * d : 0.f) + fmaf(y, al, be);
}

// CODA_A32_BN_BWD_POOLED: the layer output was max-pooled over groups of rows; only the arg-max row of a
// (group, channel) (at_max) carries the pooled gradient d
__device__ __forceinline__ float bn_bwd_pooled(float y, float d, bool at_max, float s, float h, float al, float be) {
  return ((at_max && fmaf(y, s, h) > 0.f) ? s * d : 0.f) + fmaf(y, al, be);
}

// CODA_A32_BN_BWD_POOLED_PRE: d is already [bn(y) > 0 at the arg-max row] * s * dpooled
__device__ __forceinline__ float bn_bwd_pooled_pre(float y, float d, bool at_max, float al, float be) {
  return (at_max ? d : 0.f) + fmaf(y, al, be);
}

}  // namespace a32
}  // namespace coda
