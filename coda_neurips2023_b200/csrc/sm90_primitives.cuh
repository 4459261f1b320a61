// Hopper (sm_90a) building blocks shared by the tensor-core kernels: TMA tensor-map encoding, the SM count and
// split-K scratch (host); TMA loads and stores, wgmma fences / groups and shared-memory operand descriptors (inline
// PTX).  The bf16 operand-plane format comes with it from operand_split.cuh.
#pragma once
#include <cuda.h>  // CUtensorMap types (header only; the driver entry point is fetched at run time)
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <mutex>

#include "coda_common.cuh"
#include "operand_split.cuh"
#include "wgmma_ops.cuh"

namespace coda {

// --------------------------------------------------------------------- host: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  // cuTensorMapEncodeTiled validates the global address against the CURRENT context.  An entry point that encodes a
  // map before its first runtime call can be the first CUDA call of its thread (autograd's backward worker): bind the
  // primary context to the thread once.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 16-bit matrix tiles, K contiguous: tensor [batch][rows][k] with strides (elements),
// box = [1][box_rows][64] (64 x 2 B = one 128-byte swizzle span).
inline int make_tmap_k_major_16b(CUtensorMap *map, const void *base, int is_fp16, long long k, long long rows,
                                 long long batch, long long row_stride, long long batch_stride, int box_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return CODA_EINVAL;
  cuuint64_t gdim[3] = {(cuuint64_t)k, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t gstride[2] = {(cuuint64_t)row_stride * 2, (cuuint64_t)(batch > 1 ? batch_stride : row_stride * rows) * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, is_fp16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                  const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? CODA_OK : CODA_EINVAL;
}

// fp32 matrix [rows][cols] with row stride `row_stride` (elements), box = [box_rows][box_cols], 128-byte swizzle
// (box_cols = 32: one swizzle span of fp32)
inline int make_tmap_f32_box(CUtensorMap *map, const void *base, long long cols, long long rows, long long row_stride,
                             int box_cols, int box_rows) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return CODA_EINVAL;
  cuuint64_t gdim[3] = {(cuuint64_t)cols, (cuuint64_t)rows, 1};
  cuuint64_t gstride[2] = {(cuuint64_t)row_stride * 4, (cuuint64_t)row_stride * rows * 4};
  cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void *>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? CODA_OK : CODA_EINVAL;
}

// --------------------------------------------------------------------- host: launch geometry
// SMs of the device current at the first call, kept for later calls; 132 (an H100 SXM) if the query fails.
// Persistent grids and split-K factors are sized from it.
inline int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// --------------------------------------------------------------------- host: split-K scratch
// Device scratch of the split-K GEMMs: every split writes its partial tile there and a second kernel adds the partials
// in a fixed order, so results are the same from run to run (atomic accumulation is not).  One buffer per device, grown
// outside stream capture: a captured launch must find it large enough, which the eager runs that precede a capture
// ensure.  A buffer that is outgrown is kept allocated, never freed: a CUDA graph captured while it was current still
// addresses it.  Launches that split K share the current buffer: they must not run concurrently on different streams.
inline int split_scratch(size_t floats, cudaStream_t s, float **out) {
  static std::mutex mu;
  static float *buf[64] = {};
  static size_t cap[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return CODA_EINVAL;
  std::lock_guard<std::mutex> lock(mu);
  if (cap[dev] < floats) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) return CODA_ETOOLARGE;
    // grow geometrically so that a sequence of larger launches retires few buffers
    const size_t want = floats > 2 * cap[dev] ? floats : 2 * cap[dev];
    float *p = nullptr;
    cudaError_t e = cudaMalloc(&p, want * sizeof(float));
    if (e != cudaSuccess) return (int)e;
    buf[dev] = p;
    cap[dev] = want;
  }
  *out = buf[dev];
  return CODA_OK;
}

// C[row][col] (+)= bias[col] + sum_{k < ksplit} partial[tile * ksplit + k][row - m0][col - n0], summed in split order.
// partial slots are [bm][bn] fp32 tiles; tile = (batch * tiles_m + tm) * tiles_n + tn.
static __global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float *__restrict__ partial, int ksplit, int m, int n, int batch, int bm, int bn,
                     const float *__restrict__ bias, float *__restrict__ c, long long ldc, long long c_batch_stride) {
  const long long total = (long long)batch * m * n;
  const int tiles_m = (m + bm - 1) / bm, tiles_n = (n + bn - 1) / bn;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % n);
    const long long t = i / n;
    const int row = (int)(t % m), b = (int)(t / m);
    const long long tile = ((long long)b * tiles_m + row / bm) * tiles_n + col / bn;
    const float *src = partial + (tile * ksplit) * bm * bn + (long long)(row % bm) * bn + col % bn;
    float v = bias ? __ldg(bias + col) : 0.f;
    for (int k = 0; k < ksplit; ++k) v += src[(long long)k * bm * bn];
    c[(size_t)b * c_batch_stride + (size_t)row * ldc + col] = v;
  }
}

// --------------------------------------------------------------------- device: TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 1-D bulk copy global -> shared (size and both addresses multiples of 16 bytes), completing on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// --------------------------------------------------------------------- device: warpgroup MMA
// One lane of a converged warp (the TMA-issuing warp keeps its control flow warp-uniform).
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma fences / waits
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void acc_zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}
// Move registers between warpgroups: a TMA-producer warpgroup lowers its per-thread budget so that the MMA
// warpgroups can raise theirs (every thread of the warpgroup executes the same instruction).  N: 24..256, step 8.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// named barrier over the first `threads` threads of the CTA (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// arrive on a named barrier without waiting (the other `threads - arrivals` wait on it with bar_sync)
__device__ __forceinline__ void bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// --------------------------------------------------------------------- descriptors
// K-major operand tile in shared memory, 128-byte swizzle: rows of 64 16-bit elements (128 B) stored densely,
// 8-row groups 1024 B apart (SBO), tile base 1024-byte aligned.  A 64-row slice starts 8 KB further on.
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(const void *tile) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_u32(tile) & 0x3FFFF) >> 4);  // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                             // leading byte offset: unused for swizzled K-major
  d |= (uint64_t)(1024 >> 4) << 32;                   // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                             // layout type SWIZZLE_128B
  return d;
}
// MN-major operand tile (the contraction index is the ROW index of the stored tensor): a sequence of
// [k-rows x 64 mn] boxes `lbo` bytes apart (128B-swizzled rows of 64 contiguous MN elements).  Canonical layout
// ((8,8,m),(8,k)) : ((1,8,LBO),(64,SBO)) in elements: 8-row K groups SBO = 1024 B apart, 64-wide MN groups LBO apart.
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(const void *tile, uint32_t lbo = 8192) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_u32(tile) & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo >> 4) << 16;                    // leading byte offset: next 64 MN elements
  d |= (uint64_t)(1024 >> 4) << 32;                   // stride byte offset: next 8 K rows
  d |= (uint64_t)1 << 62;                             // SWIZZLE_128B
  return d;
}

// advance the start address by `bytes` (K-major: k-steps of 32 B inside the swizzle atom; MN-major: 16 rows)
__device__ __forceinline__ uint64_t gmma_desc_advance(uint64_t desc, uint32_t bytes) { return desc + (bytes >> 4); }

// The dynamic shared-memory base rounded up to 1024 bytes, the alignment of 128B-swizzled TMA boxes and wgmma tiles
// (launches request 1024 bytes more than their layout uses).
__device__ __forceinline__ unsigned char *smem_align1024(unsigned char *smem_raw) {
  return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
}

}  // namespace coda
