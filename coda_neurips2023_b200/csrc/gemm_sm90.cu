// wgmma / TMA GEMM for H100 (sm_90a):  C[b][m][n] = sum_k A[b][m][k] * B[b][n][k]  (+ bias[n]) (ReLU)
//
// Operands are 16-bit, K-major (K contiguous) planes; fp32 inputs are first split
// into NSPLIT bf16 planes (x = hi + lo (+ lo2)) by the pack kernel below and the
// GEMM accumulates the cross products hi*hi + hi*lo + lo*hi (+ ...) in fp32
// registers, which gives fp32-class accuracy on the bf16 tensor-core path.  NSPLIT = 1
// with fp16 operands is the CLIP ViT path.
//
// Structure (persistent CTAs, 128 x BN output tiles, 288 threads):
//   warp 8        : TMA producer   (cp.async.bulk.tensor -> 128B-swizzled smem stages)
//   warps 0..7    : two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: wgmma.mma_async from the
//                   shared-memory stages into register accumulators, then +bias / activation -> global
// Split-K (long contractions, few output tiles): each split stores its partial tile in a scratch slot and
// splitk_reduce_kernel adds the slots in split order -- the result does not depend on the order the CTAs finish in.
// C-ABI in include/coda_gemm.h.
#include "../../include/coda_gemm.h"
#include "sm90_primitives.cuh"

using namespace coda;

namespace {

// ------------------------------------------------------------------ pack (fp32 -> bf16 planes)
// source is row-major along k (src_k_stride == 1): one thread per (row, k) element, k fastest
template <int NSPLIT>
__global__ void __launch_bounds__(256)
pack_rows_kernel(long long rows, int k, int kpad, long long src_row_stride, const float *__restrict__ src,
                 float scale, __nv_bfloat16 *__restrict__ planes, long long plane_stride) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * kpad) return;
  const long long r = idx / kpad;
  const int c = (int)(idx - r * kpad);
  const float x = c < k ? __ldg(src + r * src_row_stride + c) * scale : 0.f;
  split_store<NSPLIT>(x, planes + idx, (size_t)plane_stride);
}

// same, four consecutive k per thread (k % 4 == 0, 16-byte aligned rows): one 16-byte load, one 8-byte store per plane
template <int NSPLIT>
__global__ void __launch_bounds__(256)
pack_rows_vec4_kernel(long long rows, int k, int kpad, long long src_row_stride, const float *__restrict__ src,
                      float scale, __nv_bfloat16 *__restrict__ planes, long long plane_stride) {
  const int kq = kpad >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * kq) return;
  const long long r = idx / kq;
  const int c = (int)(idx - r * kq) * 4;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < k) v = __ldg(reinterpret_cast<const float4 *>(src + r * src_row_stride + c));
  split_store4<NSPLIT>(make_float4(v.x * scale, v.y * scale, v.z * scale, v.w * scale), planes + r * kpad + c,
                       (size_t)plane_stride);
}

// source is contiguous along rows (src_row_stride == 1, "transposed" operand): 32x32 smem transpose
template <int NSPLIT>
__global__ void __launch_bounds__(256)
pack_transposed_kernel(long long rows, int k, int kpad, long long src_k_stride, const float *__restrict__ src,
                       float scale, __nv_bfloat16 *__restrict__ planes, long long plane_stride) {
  __shared__ float tile[32][33];
  const long long r0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const long long r = r0 + tx;
    tile[i][tx] = (c < k && r < rows) ? __ldg(src + (long long)c * src_k_stride + r) * scale : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const long long r = r0 + i;
    const int c = c0 + tx;
    if (r < rows && c < kpad) split_store<NSPLIT>(tile[tx][i], planes + r * kpad + c, (size_t)plane_stride);
  }
}

// ------------------------------------------------------------------ GEMM
constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 2 B = one 128-byte swizzle span
constexpr int GEMM_THREADS = 288;   // warps 0-7: two consumer warpgroups (64 rows each), warp 8: TMA producer

struct GemmMaps {
  CUtensorMap a[3];
  CUtensorMap b[3];
};

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return fmaxf(x, 0.f);
  if (act == 2) return __fdividef(x, 1.0f + __expf(-1.702f * x));
  return x;
}

// MN = false: C = A B^T with K-contiguous operands ("NT").
// MN = true : both operands are stored with the contraction index as the ROW index (A planes
//             [kc][m], B planes [kc][n]) -- the weight-gradient form dW = dY^T X, which then needs no
//             transposed copies of dY and X.
template <int NSPLIT, int BN, int STAGES, bool FP16, bool MN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_nt_kernel(const __grid_constant__ GemmMaps maps, int m, int n, int kpad, int b_batched, int ksplit, int batch_n,
               const float *__restrict__ bias_in, int act, int out_half, void *__restrict__ c_void, long long ldc,
               long long c_batch_stride, const void *__restrict__ residual, long long ldr, float *__restrict__ partial) {
  // PERSISTENT: each CTA walks work items w = blockIdx.x, blockIdx.x + gridDim.x, ...;  a work item is
  // (m-tile, n-tile, batch, k-split).  The producer runs ahead into the next work item while the consumer
  // warpgroups drain their accumulators.
  constexpr int A_TILE = BM * BK * 2;
  constexpr int B_TILE = BN * BK * 2;
  constexpr int STAGE = NSPLIT * (A_TILE + B_TILE);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = smem_align1024(smem_raw);
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (m + BM - 1) / BM, tiles_n = (n + BN - 1) / BN;
  const long long nwork = (long long)tiles_m * tiles_n * batch_n * ksplit;
  const int nkb_total = kpad / BK;
  const int per = (nkb_total + ksplit - 1) / ksplit;

  // work item -> coordinates.  The CTAs that run concurrently should share operand tiles in L2: with few
  // n-tiles (skinny weights, the step's shapes) n runs fastest, so the n-tiles of one m-tile are in flight
  // together and the A rows are fetched from HBM once; with more n-tiles than m-tiles the roles swap.
  const bool n_fast = tiles_n <= tiles_m;
  auto decode = [&](long long w, int &m0, int &n0, int &batch, int &ks) {
    int tm, tn;
    if (n_fast) {
      tn = (int)(w % tiles_n); w /= tiles_n;
      tm = (int)(w % tiles_m); w /= tiles_m;
    } else {
      tm = (int)(w % tiles_m); w /= tiles_m;
      tn = (int)(w % tiles_n); w /= tiles_n;
    }
    ks = (int)(w % ksplit);
    batch = (int)(w / ksplit);
    m0 = tm * BM; n0 = tn * BN;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer (warp-uniform control flow; one elected lane issues the copies) =====
    if (lane == 0) {
#pragma unroll
      for (int p = 0; p < NSPLIT; ++p) { prefetch_tmap(&maps.a[p]); prefetch_tmap(&maps.b[p]); }
    }
    uint32_t it = 0;  // running k-block counter across work items -> stage / phase
    for (long long w = blockIdx.x; w < nwork; w += gridDim.x) {
      int m0, n0, batch, ks;
      decode(w, m0, n0, batch, ks);
      const int kb0 = ks * per, nkb = max(0, min(per, nkb_total - kb0));
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE);
          unsigned char *st = smem + (size_t)s * STAGE;
#pragma unroll
          for (int p = 0; p < NSPLIT; ++p) {
            if (!MN) {
              tma_load_3d(st + p * A_TILE, &maps.a[p], &full_bar[s], (kb0 + kb) * BK, m0, batch);
              tma_load_3d(st + NSPLIT * A_TILE + p * B_TILE, &maps.b[p], &full_bar[s], (kb0 + kb) * BK, n0,
                          b_batched ? batch : 0);
            } else {
              // [64 contraction rows x 64 mn] boxes, one per 64-wide slab of the tile
#pragma unroll
              for (int g = 0; g < BM / 64; ++g)
                tma_load_3d(st + p * A_TILE + g * 8192, &maps.a[p], &full_bar[s], m0 + g * 64, (kb0 + kb) * BK, batch);
#pragma unroll
              for (int g = 0; g < BN / 64; ++g)
                tma_load_3d(st + NSPLIT * A_TILE + p * B_TILE + g * 8192, &maps.b[p], &full_bar[s], n0 + g * 64,
                            (kb0 + kb) * BK, b_batched ? batch : 0);
            }
          }
        }
        __syncwarp();
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns rows [64 wg, +64) of every tile; accumulator in registers =====
  const int wg = warp >> 2, wl = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  float acc[BN / 2];
  uint32_t it = 0;
  for (long long w = blockIdx.x; w < nwork; w += gridDim.x) {
    int m0, n0, batch, ks;
    decode(w, m0, n0, batch, ks);
    const int kb0 = ks * per, nkb = max(0, min(per, nkb_total - kb0));
    if (nkb == 0) acc_zero(acc);   // (the launcher leaves no split empty; a slot is never left unwritten)
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1u);
      unsigned char *st = smem + (size_t)s * STAGE;
      acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < n_products(NSPLIT); ++p) {
        // the warpgroup's 64-row slice: +8 KB in both layouts (64 K-major rows, or the second [64 x 64] MN box)
        const void *at = st + prod_a(NSPLIT, p) * A_TILE + wg * 8192, *bt = st + NSPLIT * A_TILE + prod_b(NSPLIT, p) * B_TILE;
        const uint64_t ad = MN ? gmma_desc_mn_sw128(at) : gmma_desc_k_sw128(at);
        const uint64_t bd = MN ? gmma_desc_mn_sw128(bt) : gmma_desc_k_sw128(bt);
        constexpr uint32_t KSTEP = MN ? 16 * 128 : 32;  // bytes per 16-deep k-step
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk)
          Wgmma<BN, FP16>::template ss<MN ? 1 : 0, MN ? 1 : 0>(acc, gmma_desc_advance(ad, kk * KSTEP),
                                                                gmma_desc_advance(bd, kk * KSTEP), (kb | p | kk) != 0);
      }
      wgmma_commit();
      // the previous k-block's MMAs are complete: release its stage (one arrival per warpgroup)
      wgmma_wait<1>();
      acc_fence(acc);
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (nkb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);

    if (ksplit > 1) {
      // split-K: the raw partial tile goes to its scratch slot; splitk_reduce_kernel adds the slots in split order
      const long long tile = (long long)batch * tiles_m * tiles_n + (long long)(m0 / BM) * tiles_n + n0 / BN;
      float *slot = partial + (tile * ksplit + ks) * (BM * BN);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float *prow = slot + (size_t)(wg * 64 + wl * 16 + g + 8 * i) * BN;
#pragma unroll
        for (int c = 0; c < BN / 8; ++c)
          *reinterpret_cast<float2 *>(prow + c * 8 + 2 * t) = make_float2(acc[c * 4 + i * 2], acc[c * 4 + i * 2 + 1]);
      }
      continue;
    }

    // ===== epilogue: registers -> (+bias, activation, residual) -> global =====
    const float *bias = bias_in;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = m0 + wg * 64 + wl * 16 + g + 8 * i;
      if (row >= m) continue;
      float *crow = reinterpret_cast<float *>(c_void) + (size_t)batch * c_batch_stride + (size_t)row * ldc;
      __half *hrow = reinterpret_cast<__half *>(c_void) + (size_t)batch * c_batch_stride + (size_t)row * ldc;
      const __half *rrow = residual ? reinterpret_cast<const __half *>(residual) + (size_t)row * ldr : nullptr;
#pragma unroll
      for (int c = 0; c < BN / 8; ++c) {
        const int col = n0 + c * 8 + 2 * t;
        if (col >= n) continue;
        const bool pair = col + 1 < n;
        float v0 = acc[c * 4 + i * 2], v1 = acc[c * 4 + i * 2 + 1];
        if (bias) {
          v0 += __ldg(bias + col);
          if (pair) v1 += __ldg(bias + col + 1);
        }
        v0 = apply_act(v0, act);
        v1 = apply_act(v1, act);
        if (rrow) {
          v0 += __half2float(rrow[col]);
          if (pair) v1 += __half2float(rrow[col + 1]);
        }
        if (out_half) {
          if (pair && ((reinterpret_cast<uintptr_t>(hrow + col) & 3) == 0)) {
            *reinterpret_cast<__half2 *>(hrow + col) = __floats2half2_rn(v0, v1);
          } else {
            hrow[col] = __float2half_rn(v0);
            if (pair) hrow[col + 1] = __float2half_rn(v1);
          }
        } else if (pair && ((reinterpret_cast<uintptr_t>(crow + col) & 7) == 0)) {
          *reinterpret_cast<float2 *>(crow + col) = make_float2(v0, v1);
        } else {
          crow[col] = v0;
          if (pair) crow[col + 1] = v1;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ fp16 ping-pong GEMM (the CLIP tower's shapes)
// C = epilogue(A B^T) with one fp16 plane per operand, batch 1, fp16 output, n % BN == 0.  384 threads:
//   warpgroup 2    : TMA producer (setmaxnreg 40; one elected lane of its first warp issues the copies)
//   warpgroups 0, 1: consumers (setmaxnreg 232).  Warpgroup c owns whole 128 x BN tiles: the CTA's tiles
//                    j = c, c + 2, ... of its persistent work list, rows [0, 64) and [64, 128) in two accumulators.
// ptxas allocates the whole kernel within the 168 registers of the launch bound: BN = 128 (128 accumulator registers)
// fits with no spills, BN = 192 spills.
// The producer fills one stage ring in tile order; each stage is consumed (and released) by the owner of its tile.
// The two consumers issue their main loops in turn: warpgroup c starts tile j once warpgroup c ^ 1 has issued the last
// wgmma of tile j - 1 (named barrier 1 + c).  So one warpgroup's epilogue runs while the other's wgmmas keep the tensor
// pipe busy.  Every element sums its k-blocks and k16 steps in the same order as gemm_nt_kernel, then takes the same
// epilogue and one fp16 rounding: C has the same bits.
constexpr int PP_THREADS = 384;
constexpr int PP_PRODUCER_REGS = 40, PP_MMA_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 K registers
enum PpEpilogue { PP_NONE = 0, PP_BIAS = 1, PP_BIAS_GELU = 2, PP_BIAS_RES = 3 };

template <int BN, int STAGES, int EPI>
__global__ void __launch_bounds__(PP_THREADS, 1)
gemm_f16_pp_kernel(const __grid_constant__ GemmMaps maps, int m, int n, int nkb, const float *__restrict__ bias,
                   const __half *__restrict__ residual, long long ldr, __half *__restrict__ c, long long ldc) {
  constexpr int A_TILE = BM * BK * 2;
  constexpr int STAGE = A_TILE + BN * BK * 2;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = smem_align1024(smem_raw);
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (m + BM - 1) / BM, tiles_n = n / BN;
  const int ntiles = tiles_m * tiles_n;
  const bool n_fast = tiles_n <= tiles_m;   // the tile order of gemm_nt_kernel
  auto decode = [&](int w, int &m0, int &n0) {
    const int tm = n_fast ? w / tiles_n : w % tiles_m, tn = n_fast ? w % tiles_n : w / tiles_m;
    m0 = tm * BM; n0 = tn * BN;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===== TMA producer warpgroup =====
    setmaxnreg_dec<PP_PRODUCER_REGS>();
    if (warp != 8) return;
    if (lane == 0) { prefetch_tmap(&maps.a[0]); prefetch_tmap(&maps.b[0]); }
    uint32_t it = 0;
    for (int w = blockIdx.x; w < ntiles; w += gridDim.x) {
      int m0, n0;
      decode(w, m0, n0);
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(&empty_bar[s], ((it / STAGES) & 1u) ^ 1u);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE);
          unsigned char *st = smem + (size_t)s * STAGE;
          tma_load_3d(st, &maps.a[0], &full_bar[s], kb * BK, m0, 0);
          tma_load_3d(st + A_TILE, &maps.b[0], &full_bar[s], kb * BK, n0, 0);
        }
        __syncwarp();
      }
    }
    return;
  }
  setmaxnreg_inc<PP_MMA_REGS>();

  // ===== consumers: warpgroup wg owns every other tile of the CTA; accumulators for rows [0, 64) and [64, 128) =====
  const int wg = warp >> 2, wl = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  float acc[2][BN / 2];
  // ring position of the tile's first k-block: the CTA's j-th tile starts at j * nkb
  uint32_t it = (uint32_t)(wg * nkb);
  for (int w = blockIdx.x + wg * gridDim.x; w < ntiles; w += 2 * gridDim.x, it += 2 * nkb) {
    int m0, n0;
    decode(w, m0, n0);
    const bool other_next = w + (int)gridDim.x < ntiles;   // the other warpgroup has the CTA's next tile
    // wait for the turn: the other warpgroup has issued all wgmmas of the CTA's previous tile
    if (wg == 1 || w != (int)blockIdx.x) bar_sync(1 + wg, 256);
    for (int kb = 0; kb < nkb; ++kb) {
      const uint32_t i = it + kb;
      const int s = i % STAGES;
      mbar_wait(&full_bar[s], (i / STAGES) & 1u);
      unsigned char *st = smem + (size_t)s * STAGE;
      acc_fence(acc[0]);
      acc_fence(acc[1]);
      wgmma_fence();
      const uint64_t ad = gmma_desc_k_sw128(st), bd = gmma_desc_k_sw128(st + A_TILE);
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        const uint64_t b = gmma_desc_advance(bd, kk * 32);
        Wgmma<BN, true>::template ss<0, 0>(acc[0], gmma_desc_advance(ad, kk * 32), b, (kb | kk) != 0);
        Wgmma<BN, true>::template ss<0, 0>(acc[1], gmma_desc_advance(ad, 8192 + kk * 32), b, (kb | kk) != 0);
      }
      wgmma_commit();
      if (kb == nkb - 1 && other_next) bar_arrive(1 + (wg ^ 1), 256);   // hand the turn over
      // the previous k-block's MMAs are complete: release its stage
      wgmma_wait<1>();
      acc_fence(acc[0]);
      acc_fence(acc[1]);
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
    }

    // bias of the thread's column pairs, read once per tile while the last k-block's MMAs run
    float2 bv[BN / 8];
    if (EPI != PP_NONE) {
#pragma unroll
      for (int cc = 0; cc < BN / 8; ++cc) bv[cc] = __ldg(reinterpret_cast<const float2 *>(bias + n0 + cc * 8 + 2 * t));
    }
    wgmma_wait<0>();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it + nkb - 1) % STAGES]);

    // ===== epilogue: fp32 accumulator + bias, activation, + residual, one fp16 rounding =====
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = m0 + h * 64 + wl * 16 + g + 8 * r;
        if (row >= m) continue;
        __half *crow = c + (size_t)row * ldc + n0 + 2 * t;
        const __half *rrow = EPI == PP_BIAS_RES ? residual + (size_t)row * ldr + n0 + 2 * t : nullptr;
#pragma unroll
        for (int cc = 0; cc < BN / 8; ++cc) {
          float v0 = acc[h][cc * 4 + r * 2], v1 = acc[h][cc * 4 + r * 2 + 1];
          if (EPI != PP_NONE) { v0 += bv[cc].x; v1 += bv[cc].y; }
          if (EPI == PP_BIAS_GELU) { v0 = apply_act(v0, 2); v1 = apply_act(v1, 2); }
          if (EPI == PP_BIAS_RES) {
            const __half2 rv = *reinterpret_cast<const __half2 *>(rrow + cc * 8);
            v0 += __low2float(rv);
            v1 += __high2float(rv);
          }
          *reinterpret_cast<__half2 *>(crow + cc * 8) = __floats2half2_rn(v0, v1);
        }
      }
    }
  }
}

template <int NSPLIT, int BN, int STAGES, bool FP16, bool MN = false>
int launch_gemm(const GemmMaps &maps, int batch, int m, int n, int kpad, int b_batched, const float *bias, int relu,
                void *c_out, long long ldc, long long c_batch_stride, cudaStream_t s, int out_half = 0,
                const void *residual = nullptr, long long ldr = 0) {
  float *c = reinterpret_cast<float *>(c_out);
  const int sms = sm_count();
  // split-K when the output has few tiles but the contraction is long (weight gradients)
  const long long tiles = (long long)((m + BM - 1) / BM) * ((n + BN - 1) / BN) * batch;
  const int nkb_total = kpad / BK;
  int ksplit = 1;
  if (!relu && !out_half && tiles < sms && nkb_total >= 32) {
    ksplit = (int)((2 * sms + tiles - 1) / tiles);
    if (ksplit > nkb_total / 8) ksplit = nkb_total / 8;
    if (ksplit < 1) ksplit = 1;
    // as many splits as the k-blocks per split need: none is left empty
    const int per = (nkb_total + ksplit - 1) / ksplit;
    ksplit = (nkb_total + per - 1) / per;
  }
  if (residual && (!FP16 || !out_half || batch != 1 || (ldr & 7) != 0 || ((uintptr_t)residual & 15) != 0))
    return CODA_EINVAL;   // the fused residual exists on the fp16-output path only
  float *partial = nullptr;
  if (ksplit > 1) {
    const int st = split_scratch((size_t)tiles * ksplit * BM * BN, s, &partial);
    if (st != CODA_OK) return st;
  }
  constexpr size_t smem = (size_t)STAGES * NSPLIT * (BM * BK * 2 + BN * BK * 2) + 1024;
  static_assert(smem <= 227 * 1024, "smem budget");
  constexpr auto kern = gemm_nt_kernel<NSPLIT, BN, STAGES, FP16, MN>;
  if (const int st = raise_smem_limit<kern>((int)smem)) return st;
  const long long nwork = tiles * ksplit;
  const unsigned grid = (unsigned)(nwork < sms ? nwork : sms);
  kern<<<grid, GEMM_THREADS, smem, s>>>(maps, m, n, kpad, b_batched, ksplit, batch, bias, relu, out_half, c_out, ldc,
                                        c_batch_stride, residual, ldr, partial);
  if (ksplit > 1) {
    const long long total = (long long)batch * m * n;
    const long long blocks = (total + 255) / 256;
    splitk_reduce_kernel<<<(unsigned)(blocks < 8 * sms ? blocks : 8 * sms), 256, 0, s>>>(partial, ksplit, m, n, batch, BM,
                                                                                          BN, bias, c, ldc, c_batch_stride);
  }
  return launch_status();
}

template <int BN, int STAGES, int EPI>
int launch_gemm_f16_pp(const GemmMaps &maps, int m, int n, int kpad, const float *bias, const void *residual,
                       long long ldr, void *c, long long ldc, cudaStream_t s) {
  constexpr size_t smem = (size_t)STAGES * (BM * BK * 2 + BN * BK * 2) + 1024;
  static_assert(smem <= 227 * 1024, "smem budget");
  constexpr auto kern = gemm_f16_pp_kernel<BN, STAGES, EPI>;
  if (const int st = raise_smem_limit<kern>((int)smem)) return st;
  const int sms = sm_count();
  const int tiles = (m + BM - 1) / BM * (n / BN);
  kern<<<(unsigned)(tiles < sms ? tiles : sms), PP_THREADS, smem, s>>>(
      maps, m, n, kpad / BK, bias, reinterpret_cast<const __half *>(residual), ldr, reinterpret_cast<__half *>(c), ldc);
  return launch_status();
}

}  // namespace

extern "C" {

int coda_pack_split_bf16_strided(long long rows, int k, int kpad, long long src_row_stride,
                                 long long src_k_stride, const float *src, float scale, int nsplit, void *planes,
                                 long long plane_stride, void *stream) {
  if (rows < 0 || k < 0 || kpad < k || kpad % 64 != 0 || nsplit < 1 || nsplit > 3) return CODA_EINVAL;
  if (rows == 0 || kpad == 0) return CODA_OK;
  if (!src || !planes) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  __nv_bfloat16 *out = (__nv_bfloat16 *)planes;
  if ((src_k_stride == 1 || k <= 1) && k % 4 == 0 && src_row_stride % 4 == 0 && ((uintptr_t)src & 15) == 0 &&
      plane_stride % 4 == 0 && ((uintptr_t)out & 7) == 0) {
    const long long total = rows * (kpad / 4);
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (nsplit == 1) pack_rows_vec4_kernel<1><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
    else if (nsplit == 2) pack_rows_vec4_kernel<2><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
    else pack_rows_vec4_kernel<3><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
  } else if (src_k_stride == 1 || k <= 1) {
    const long long total = rows * kpad;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (nsplit == 1) pack_rows_kernel<1><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
    else if (nsplit == 2) pack_rows_kernel<2><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
    else pack_rows_kernel<3><<<grid, 256, 0, s>>>(rows, k, kpad, src_row_stride, src, scale, out, plane_stride);
  } else if (src_row_stride == 1) {
    const dim3 grid((unsigned)((rows + 31) / 32), (kpad + 31) / 32);
    if (grid.y > 65535) return CODA_ETOOLARGE;
    if (nsplit == 1) pack_transposed_kernel<1><<<grid, 256, 0, s>>>(rows, k, kpad, src_k_stride, src, scale, out, plane_stride);
    else if (nsplit == 2) pack_transposed_kernel<2><<<grid, 256, 0, s>>>(rows, k, kpad, src_k_stride, src, scale, out, plane_stride);
    else pack_transposed_kernel<3><<<grid, 256, 0, s>>>(rows, k, kpad, src_k_stride, src, scale, out, plane_stride);
  } else {
    return CODA_EINVAL;  // one of the two strides must be 1
  }
  return launch_status();
}

int coda_pack_split_bf16(long long rows, int k, int kpad, long long src_row_stride, long long src_k_stride,
                         const float *src, float scale, int nsplit, void *planes, void *stream) {
  return coda_pack_split_bf16_strided(rows, k, kpad, src_row_stride, src_k_stride, src, scale, nsplit, planes,
                                      rows * kpad, stream);
}

int coda_gemm_nt(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                 long long a_plane_stride, long long a_batch_stride, const void *b, long long b_plane_stride,
                 long long b_batch_stride, const float *bias, int relu, float *c, long long ldc,
                 long long c_batch_stride, void *stream) {
  return coda_gemm_nt_ex(nsplit, is_fp16, batch, m, n, kpad, a, a_plane_stride, a_batch_stride, b, b_plane_stride,
                         b_batch_stride, bias, relu, 0, c, ldc, c_batch_stride, stream);
}

int coda_gemm_nt_ex(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                    long long a_plane_stride, long long a_batch_stride, const void *b, long long b_plane_stride,
                    long long b_batch_stride, const float *bias, int relu, int out_half, void *c, long long ldc,
                    long long c_batch_stride, void *stream) {
  return coda_gemm_nt_res(nsplit, is_fp16, batch, m, n, kpad, a, a_plane_stride, a_batch_stride, b, b_plane_stride,
                          b_batch_stride, bias, relu, out_half, nullptr, 0, c, ldc, c_batch_stride, stream);
}

int coda_gemm_nt_res(int nsplit, int is_fp16, int batch, int m, int n, int kpad, const void *a,
                     long long a_plane_stride, long long a_batch_stride, const void *b, long long b_plane_stride,
                     long long b_batch_stride, const float *bias, int relu, int out_half, const void *residual,
                     long long ldr, void *c, long long ldc, long long c_batch_stride, void *stream) {
  if (nsplit < 1 || nsplit > 3 || batch < 0 || m < 0 || n < 0 || kpad < 0 || kpad % 64 != 0) return CODA_EINVAL;
  if (is_fp16 && nsplit != 1) return CODA_EINVAL;
  if (batch == 0 || m == 0 || n == 0) return CODA_OK;
  if (!a || !b || !c || kpad == 0 || batch > 65535) return CODA_EINVAL;
  // fp16 tower GEMMs with wide outputs: a 128 x 256 tile moves 48 KB per k-block for twice the flops of a 128 x 128
  // tile (32 KB).  N = 768 (attention / MLP output projections of the ViT) takes 192-wide tiles: more flops per
  // byte than 128-wide ones, and a 768-wide row is still an exact number of tiles.
  // The ping-pong kernel takes fp16-output calls with the epilogues the CLIP tower uses, 128-wide tiles that divide n,
  // 16-byte aligned outputs / residual rows, and at least two tiles per SM: with fewer, one warpgroup per SM would sit
  // idle and the 288-thread kernel, whose warpgroups share each tile, is the better fit.
  constexpr int PP_BN = 128;
  const int pp_epi = !bias ? (relu == 0 && !residual ? PP_NONE : -1)
                     : relu == 0 ? (residual ? PP_BIAS_RES : PP_BIAS)
                     : (relu == 2 && !residual) ? PP_BIAS_GELU : -1;
  const long long pp_tiles = (long long)((m + BM - 1) / BM) * (n / PP_BN);   // int tile indices in the kernel
  const bool pp = is_fp16 && out_half && batch == 1 && pp_epi >= 0 && n % PP_BN == 0 &&
                  pp_tiles >= 2LL * sm_count() && pp_tiles <= INT_MAX && ldc % 8 == 0 &&
                  ((uintptr_t)c & 15) == 0 && ((uintptr_t)bias & 7) == 0 &&
                  (!residual || (ldr % 8 == 0 && ((uintptr_t)residual & 15) == 0));
  const int bn = pp ? PP_BN
                 : n <= 64 ? 64
                 : (is_fp16 && n % 256 == 0 && n >= 1536) ? 256
                 : (is_fp16 && n % 192 == 0 && n >= 384)  ? 192
                                                          : 128;
  GemmMaps maps;
  const char *ap = (const char *)a, *bp = (const char *)b;
  for (int p = 0; p < nsplit; ++p) {
    int st = make_tmap_k_major_16b(&maps.a[p], ap + (size_t)p * a_plane_stride * 2, is_fp16, kpad, m, batch, kpad,
                                   a_batch_stride, BM);
    if (st != CODA_OK) return st;
    st = make_tmap_k_major_16b(&maps.b[p], bp + (size_t)p * b_plane_stride * 2, is_fp16, kpad, n,
                               b_batch_stride ? batch : 1, kpad, b_batch_stride, bn);
    if (st != CODA_OK) return st;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int bb = b_batch_stride ? 1 : 0;
#define CODA_GEMM(NS, BN_, ST, F16) \
  return launch_gemm<NS, BN_, ST, F16>(maps, batch, m, n, kpad, bb, bias, relu, c, ldc, c_batch_stride, s, out_half, \
                                       residual, ldr)
  if (pp) {
#define CODA_GEMM_PP(EPI) \
  return launch_gemm_f16_pp<PP_BN, 6, EPI>(maps, m, n, kpad, bias, residual, ldr, c, ldc, s)
    if (pp_epi == PP_NONE) CODA_GEMM_PP(PP_NONE);
    if (pp_epi == PP_BIAS) CODA_GEMM_PP(PP_BIAS);
    if (pp_epi == PP_BIAS_GELU) CODA_GEMM_PP(PP_BIAS_GELU);
    CODA_GEMM_PP(PP_BIAS_RES);
#undef CODA_GEMM_PP
  }
  if (is_fp16) {
    if (bn == 64) CODA_GEMM(1, 64, 6, true);
    if (bn == 256) CODA_GEMM(1, 256, 4, true);
    if (bn == 192) CODA_GEMM(1, 192, 5, true);
    CODA_GEMM(1, 128, 6, true);
  }
  if (nsplit == 1) {
    if (bn == 64) CODA_GEMM(1, 64, 6, false);
    CODA_GEMM(1, 128, 6, false);
  }
  if (nsplit == 2) {
    if (bn == 64) CODA_GEMM(2, 64, 4, false);
    CODA_GEMM(2, 128, 3, false);
  }
  if (bn == 64) CODA_GEMM(3, 64, 2, false);
  CODA_GEMM(3, 128, 2, false);
#undef CODA_GEMM
}


int coda_gemm_tn(int nsplit, int mc, int m, int n, const void *a, long long a_plane_stride, int lda,
                 const void *b, long long b_plane_stride, int ldb, float *c, long long ldc, void *stream) {
  // C[m][n] = sum_r A[r][m] * B[r][n], r < mc;  A planes [nsplit][mc][lda], B planes [nsplit][mc][ldb]
  if (nsplit < 1 || nsplit > 3 || mc < 0 || m < 0 || n < 0 || lda % 64 != 0 || ldb % 64 != 0) return CODA_EINVAL;
  if (m == 0 || n == 0) return CODA_OK;
  if (!a || !b || !c || mc == 0 || lda < m || ldb < n) return CODA_EINVAL;
  const int bn = n <= 64 ? 64 : 128;
  GemmMaps maps;
  const char *ap = (const char *)a, *bp = (const char *)b;
  for (int p = 0; p < nsplit; ++p) {
    // tensors [1][mc rows][lda cols]; box = [64 rows][64 cols]
    int st = make_tmap_k_major_16b(&maps.a[p], ap + (size_t)p * a_plane_stride * 2, 0, lda, mc, 1, lda, 0, 64);
    if (st != CODA_OK) return st;
    st = make_tmap_k_major_16b(&maps.b[p], bp + (size_t)p * b_plane_stride * 2, 0, ldb, mc, 1, ldb, 0, 64);
    if (st != CODA_OK) return st;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int kpad = (mc + 63) / 64 * 64;  // contraction length in 64-row blocks (rows >= mc read as zero)
#define CODA_GEMM_TN(NS, BN_, ST) \
  return launch_gemm<NS, BN_, ST, false, true>(maps, 1, m, n, kpad, 0, nullptr, 0, c, ldc, 0, s)
  if (nsplit == 1) { if (bn == 64) CODA_GEMM_TN(1, 64, 6); CODA_GEMM_TN(1, 128, 6); }
  if (nsplit == 2) { if (bn == 64) CODA_GEMM_TN(2, 64, 4); CODA_GEMM_TN(2, 128, 3); }
  if (bn == 64) CODA_GEMM_TN(3, 64, 2);
  CODA_GEMM_TN(3, 128, 2);
#undef CODA_GEMM_TN
}

}  // extern "C"
