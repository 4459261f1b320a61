// Test-time classification of predicted boxes by their CLIP crop features (include/coda_image.h
// coda_clip_classify).  A CTA owns R (scene, query) rows: their normalised features sit in shared memory in fp64,
// each warp walks a strided share of the classes and forms the R dot products of one text row per pass (one
// coalesced read of the text row serves all R rows), the R x c logits stay in shared memory in fp64, and warp r
// finishes row r's softmax.  Every reduction has a fixed shape, so the bits do not depend on scheduling.
#include <math.h>

#include "../../include/coda_image.h"
#include "coda_common.cuh"

using namespace coda;

namespace {

constexpr int D = 512;             // CLIP ViT-B embedding width
constexpr int PER_LANE = D / 32;
constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// R rows per CTA; R == WARPS (warp r owns row r) or R == 1 (warp 0 owns the row, for large c)
template <int R>
__global__ void __launch_bounds__(THREADS) clip_classify_kernel(long long rows, int n, int c,
                                                                const float *__restrict__ feats,
                                                                const float *__restrict__ text,
                                                                const float *__restrict__ scale,
                                                                const int *__restrict__ row_map,
                                                                float *__restrict__ prob, float *__restrict__ logits) {
  extern __shared__ double smem[];
  double *f = smem;                  // R x D normalised features
  double *z = smem + R * D;          // R x c logits
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row0 = (long long)blockIdx.x * R;

  // 1. the feature of each row, divided by its norm (zeros for a skipped row)
  int usable = 0;
  if (warp < R) {
    const long long row = row0 + warp;
    int m = -1;
    if (row < rows) {
      m = row_map[row];
      if (m >= n) m = -1;
    }
    double v[PER_LANE];
    double ss = 0.0;
#pragma unroll
    for (int k = 0; k < PER_LANE; ++k) {
      v[k] = m >= 0 ? (double)feats[(long long)m * D + lane + 32 * k] : 0.0;
      ss = fma(v[k], v[k], ss);
    }
    ss = warp_sum(ss);
    const double inv = m >= 0 ? 1.0 / sqrt(ss) : 0.0;
#pragma unroll
    for (int k = 0; k < PER_LANE; ++k) f[warp * D + lane + 32 * k] = v[k] * inv;
    usable = m >= 0;
  }
  const int any = __syncthreads_or(usable);

  // 2. logits: warp w takes classes w, w + WARPS, ...
  if (any) {
    const double s = (double)scale[0];
    for (int cls = warp; cls < c; cls += WARPS) {
      double t[PER_LANE];
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) t[k] = (double)text[(long long)cls * D + lane + 32 * k];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < PER_LANE; ++k) acc = fma(f[r * D + lane + 32 * k], t[k], acc);
        acc = warp_sum(acc);
        if (lane == 0) z[r * c + cls] = s * acc;
      }
    }
  }
  __syncthreads();

  // 3. warp r: softmax of row r, or zeros; the logits output is zero throughout
  if (warp < R) {
    const long long row = row0 + warp;
    if (row >= rows) return;
    float *p = prob + row * c;
    if (logits)
      for (int j = lane; j < c; j += 32) logits[row * c + j] = 0.0f;
    if (!usable) {
      for (int j = lane; j < c; j += 32) p[j] = 0.0f;
      return;
    }
    const double *zr = z + warp * c;
    double mx = -INFINITY;
    for (int j = lane; j < c; j += 32) mx = fmax(mx, zr[j]);
    mx = warp_max(mx);
    double sum = 0.0;
    for (int j = lane; j < c; j += 32) sum += exp(zr[j] - mx);
    sum = warp_sum(sum);
    const double inv = 1.0 / sum;
    for (int j = lane; j < c; j += 32) p[j] = (float)(exp(zr[j] - mx) * inv);
  }
}

constexpr int MAX_SMEM = 227 * 1024;

template <int R>
size_t smem_bytes(int c) {
  return sizeof(double) * ((size_t)R * D + (size_t)R * c);
}

template <int R>
int launch(long long rows, int n, int c, const float *feats, const float *text, const float *scale,
           const int *row_map, float *prob, float *logits, cudaStream_t stream) {
  const size_t bytes = smem_bytes<R>(c);
  // per device, so set on every launch that needs more than the default 48 KB
  if (bytes > 48 * 1024 &&
      cudaFuncSetAttribute(clip_classify_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) !=
          cudaSuccess)
    return launch_status();
  const long long blocks = (rows + R - 1) / R;
  clip_classify_kernel<R><<<(unsigned)blocks, THREADS, bytes, stream>>>(rows, n, c, feats, text, scale, row_map,
                                                                         prob, logits);
  return launch_status();
}

}  // namespace

extern "C" int coda_clip_classify(long long rows, int n, int c, int d, const float *feats, const float *text,
                                  const float *scale, const int *row_map, float *prob, float *logits,
                                  void *stream) {
  if (rows < 0 || n < 0 || c < 1 || d != D) return CODA_EINVAL;
  if (rows == 0) return CODA_OK;
  if (!text || !scale || !row_map || !prob || (n > 0 && !feats)) return CODA_EINVAL;
  if (rows > 0x7fffffffLL) return CODA_ETOOLARGE;
  cudaStream_t st = (cudaStream_t)stream;
  if (smem_bytes<WARPS>(c) <= (size_t)MAX_SMEM)
    return launch<WARPS>(rows, n, c, feats, text, scale, row_map, prob, logits, st);
  if (smem_bytes<1>(c) <= (size_t)MAX_SMEM)
    return launch<1>(rows, n, c, feats, text, scale, row_map, prob, logits, st);
  return CODA_ETOOLARGE;
}
