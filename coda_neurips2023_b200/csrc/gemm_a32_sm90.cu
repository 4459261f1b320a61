// wgmma GEMM whose A operand is read as FP32 ROWS and turned into bf16 operand planes INSIDE the kernel:
//
//     C[m][n] = sum_k T(A)[m][k] * B[n][k]  (+ bias[n]) (ReLU),      T = per-element prologue on A
//
// Why: the split-bf16 GEMM of gemm_sm90.cu needs its A operand as 2-3 bf16 planes in HBM -- every fp32
// activation would be written again as 6 B/element by a pack kernel and read back by the GEMM, and the BatchNorm
// between two layers of the set-abstraction MLP would cost another full read + plane write.  Here A is loaded once
// as fp32 (4 B/element, TMA, 128B-swizzled); every consumer thread reads its own A-fragment elements from the raw
// tile, applies T (identity | per-channel affine + ReLU, i.e. BatchNorm+ReLU with batch statistics folded into
// scale/shift | the BatchNorm-backward forms), splits the values into NSPLIT bf16 planes in registers and hands
// them to wgmma as the register A operand.  Only B (the weights) goes through shared-memory descriptors.
//
// Epilogue options: bias / ReLU, and per-column sum / sum-of-squares partials of the OUTPUT (the BatchNorm
// statistics of the layer just computed: no separate pass over C).
//
// Warp roles (288 threads, persistent CTAs, one per SM):
//   warp 8      TMA producer: raw fp32 A boxes -> raw ring, B plane boxes -> B ring
//   warps 0-7   two consumer warpgroups (rows [0, 64) and [64, 128) of the tile): prologue -> register A
//               fragments -> wgmma.mma_async (B from shared memory) -> register accumulators -> epilogue
// C-ABI in include/coda_gemm.h (coda_gemm_a32*).
#include "../../include/coda_gemm.h"
#include "sm90_primitives.cuh"

using namespace coda;

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int RAW_TILE = BM * BK * 4;   // 32 KB: two [128 rows x 32 fp32] SW128 boxes
constexpr int A32_THREADS = 288;

struct A32Maps {
  CUtensorMap a;      // fp32 [m][k], box [128][32]
  CUtensorMap a2;     // second fp32 input of the two-input modes (same geometry)
  CUtensorMap b[3];   // bf16 planes
};

__host__ __device__ constexpr int n_products(int ns) { return ns == 1 ? 1 : (ns == 2 ? 3 : 6); }
__host__ __device__ constexpr int prod_a(int ns, int p) {
  return ns == 1 ? 0 : ns == 2 ? (p == 0 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 2 : p == 2 ? 0 : p == 3 ? 1 : 0);
}
__host__ __device__ constexpr int prod_b(int ns, int p) {
  return ns == 1 ? 0 : ns == 2 ? (p == 1 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 0 : p == 2 ? 2 : p == 3 ? 0 : p == 4 ? 1 : 0);
}

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

struct A32Params {
  int m, n, k;             // k = logical contraction length (A columns); B planes are padded to kpad
  int mode;                // CODA_A32_*
  const float *scale;      // per-k, padded to a multiple of 64: modes 1-3 evaluate z = a * scale + shift
  const float *shift;
  const float *alpha;      // modes 2, 3 (BatchNorm backward): T = [z > 0] * scale * d + a * alpha + beta
  const float *beta;
  const float *dpooled;    // mode 3: (m / group, k) gradient of the max-pooled output
  const unsigned char *argmax;   // mode 3: (m / group, k) arg-max row within the group
  int group;               // mode 3
  const float *bias;
  int act;
  float *c;
  long long ldc;
  float *stats;            // [gridDim.x][2][n] or null
  int b_resident;          // the whole B operand of this CTA's n-tile stays in shared memory (short contractions)
};

// RAW_KB: size of the raw-fp32 staging region; it holds RAW_KB / 32 stages (one-input prologues) or RAW_KB / 64
// (the two-input BatchNorm-backward prologue).
template <int NSPLIT, int BN, int RAW_KB, int B_STAGES, bool B_MN>
__global__ void __launch_bounds__(A32_THREADS, 1)
gemm_a32_kernel(const __grid_constant__ A32Maps maps, const A32Params P) {
  constexpr int MAX_RAW = RAW_KB / 32;
  constexpr int B_TILE = BN * BK * 2;
  constexpr int B_STAGE = NSPLIT * B_TILE;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char *raw_ring = smem;
  const bool two_in = P.mode == CODA_A32_BN_BWD;
  const bool pooled = P.mode == CODA_A32_BN_BWD_POOLED || P.mode == CODA_A32_BN_BWD_POOLED_PRE;
  // pooled BatchNorm backward: each raw stage carries, after the fp32 tile, the (group, channel) gradient and
  // arg-max rows of the tile's groups for this k-block: [groups in tile][64 floats | 64 bytes]  (<= 1 KB)
  const int raw_stage_bytes = RAW_TILE * (two_in ? 2 : 1) + (pooled ? 1024 : 0);
  const uint32_t nraw = (uint32_t)((RAW_KB * 1024) / raw_stage_bytes);
  const int tile_groups = pooled ? (P.group >= BM ? 1 : BM / P.group) : 0;
  unsigned char *b_ring = smem + (size_t)RAW_KB * 1024;
  float *s_stats = reinterpret_cast<float *>(b_ring + (size_t)B_STAGES * B_STAGE);   // [8 warps][2][n] (only if P.stats)
  __shared__ __align__(8) uint64_t raw_full[MAX_RAW], raw_empty[MAX_RAW];
  __shared__ __align__(8) uint64_t b_full[B_STAGES], b_empty[B_STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = P.m, n = P.n;
  const int tiles_m = (m + BM - 1) / BM, tiles_n = (n + BN - 1) / BN;
  const long long nwork = (long long)tiles_m * tiles_n;
  const int nkb = (P.k + BK - 1) / BK;
  // n runs fastest: the n-tiles of one m-tile are in flight together on neighbouring CTAs, A comes from HBM once
  // B-resident mode: a CTA keeps ONE n-tile for its whole life (its B planes are loaded once and never leave
  // shared memory) and walks the m-tiles with stride gridDim / tiles_n.
  auto tile_at = [&](long long t, int &m0, int &n0) -> bool {
    if (P.b_resident) {
      const int per = (int)gridDim.x / tiles_n;
      const long long tm = (long long)(blockIdx.x / tiles_n) + t * per;
      if ((int)blockIdx.x >= per * tiles_n || tm >= tiles_m) return false;
      m0 = (int)tm * BM;
      n0 = (int)(blockIdx.x % tiles_n) * BN;
      return true;
    }
    const long long w = blockIdx.x + t * gridDim.x;
    if (w >= nwork) return false;
    n0 = (int)(w % tiles_n) * BN;
    m0 = (int)(w / tiles_n) * BM;
    return true;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_RAW; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], 8); }
    for (int s = 0; s < B_STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 2); }
    mbar_fence_init_cluster();
  }
  if (P.stats && warp < 8) {
    float *mine = s_stats + (size_t)warp * 2 * n;
    for (int i = lane; i < 2 * n; i += 32) mine[i] = 0.f;
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      prefetch_tmap(&maps.a);
      if (two_in) prefetch_tmap(&maps.a2);
#pragma unroll
      for (int p = 0; p < NSPLIT; ++p) prefetch_tmap(&maps.b[p]);
    }
    uint32_t it = 0;
    int m0, n0;
    auto load_b = [&](int kb, int bs) {
      unsigned char *bt = b_ring + (size_t)bs * B_STAGE;
      mbar_arrive_expect_tx(&b_full[bs], (uint32_t)B_STAGE);
#pragma unroll
      for (int p = 0; p < NSPLIT; ++p) {
        if (!B_MN) {
          tma_load_3d(bt + p * B_TILE, &maps.b[p], &b_full[bs], kb * BK, n0, 0);
        } else {
#pragma unroll
          for (int g = 0; g < BN / 64; ++g)
            tma_load_3d(bt + p * B_TILE + g * 8192, &maps.b[p], &b_full[bs], n0 + g * 64, kb * BK, 0);
        }
      }
    };
    if (P.b_resident && tile_at(0, m0, n0)) {
      if (elect_one_sync())
        for (int kb = 0; kb < nkb; ++kb) load_b(kb, kb);
      __syncwarp();
    }
    for (long long t = 0; tile_at(t, m0, n0); ++t) {
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int rs = it % nraw, bs = it % B_STAGES;
        mbar_wait(&raw_empty[rs], ((it / nraw) & 1u) ^ 1u);
        if (!P.b_resident) mbar_wait(&b_empty[bs], ((it / B_STAGES) & 1u) ^ 1u);
        if (elect_one_sync()) {
          unsigned char *rt = raw_ring + (size_t)rs * raw_stage_bytes;
          mbar_arrive_expect_tx(&raw_full[rs], (uint32_t)(RAW_TILE * (two_in ? 2 : 1) + tile_groups * 320));
          if (pooled) {
            const long long ngroups = P.m / P.group;
            for (int gt = 0; gt < tile_groups; ++gt) {
              long long g = (long long)m0 / P.group + gt;
              if (g >= ngroups) g = ngroups - 1;        // rows past m: values unused
              bulk_load_1d(rt + RAW_TILE + gt * 320, P.dpooled + g * P.k + kb * BK, 256, &raw_full[rs]);
              bulk_load_1d(rt + RAW_TILE + gt * 320 + 256, P.argmax + g * P.k + kb * BK, 64, &raw_full[rs]);
            }
          }
          tma_load_3d(rt, &maps.a, &raw_full[rs], kb * BK, m0, 0);
          tma_load_3d(rt + RAW_TILE / 2, &maps.a, &raw_full[rs], kb * BK + 32, m0, 0);
          if (two_in) {
            tma_load_3d(rt + RAW_TILE, &maps.a2, &raw_full[rs], kb * BK, m0, 0);
            tma_load_3d(rt + RAW_TILE + RAW_TILE / 2, &maps.a2, &raw_full[rs], kb * BK + 32, m0, 0);
          }
          if (!P.b_resident) load_b(kb, bs);
        }
        __syncwarp();
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns rows [64 wg, +64) of the tile =====
  const int wg = warp >> 2, wl = warp & 3;
  const int g = lane >> 2, t4 = lane & 3;
  const int rloc[2] = {wg * 64 + wl * 16 + g, wg * 64 + wl * 16 + g + 8};   // this thread's two rows of the tile
  float *my_stats = P.stats ? s_stats + (size_t)warp * 2 * n : nullptr;
  float acc[BN / 2];
  uint32_t it = 0;
  int m0, n0;
  for (long long t = 0; tile_at(t, m0, n0); ++t) {
    // pooled mode: the 16 rows of a warp lie in one group (group % 32 == 0); index of each row within it
    int pgt = 0, pgi[2] = {0, 0};
    if (pooled) {
      pgt = P.group >= BM ? 0 : rloc[0] / P.group;
#pragma unroll
      for (int i = 0; i < 2; ++i) pgi[i] = (int)(((long long)m0 + rloc[i]) % P.group);
    }
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int rs = it % nraw, bs = P.b_resident ? kb : (int)(it % B_STAGES);
      mbar_wait(&raw_full[rs], (it / nraw) & 1u);
      const unsigned char *rt = raw_ring + (size_t)rs * raw_stage_bytes;
      const int k0 = kb * BK;
      // A fragments of the four 16-deep k-steps: register q of step kk holds (row rloc[q & 1], columns
      // 16 kk + 8 (q >> 1) + 2 t4 + {0, 1})
      uint32_t af[BK / 16][NSPLIT][4];
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int row = rloc[q & 1];
          const int col = kk * 16 + (q >> 1) * 8 + 2 * t4;   // column of the k-block (even)
          const uint32_t off = (uint32_t)(col >> 5) * (RAW_TILE / 2) + (uint32_t)row * 128u +
                               ((uint32_t)(((col & 31) >> 2) ^ (row & 7)) << 4) + (uint32_t)(col & 3) * 4u;
          float2 x = *reinterpret_cast<const float2 *>(rt + off);
          const int kc = k0 + col;
          if (P.mode == CODA_A32_AFFINE_RELU) {
            const float2 s2 = __ldg(reinterpret_cast<const float2 *>(P.scale + kc));
            const float2 h2 = __ldg(reinterpret_cast<const float2 *>(P.shift + kc));
            x.x = fmaxf(fmaf(x.x, s2.x, h2.x), 0.f);
            x.y = fmaxf(fmaf(x.y, s2.y, h2.y), 0.f);
          } else if (P.mode == CODA_A32_BN_BWD) {
            // x = y (pre-BN activation), d = gradient of relu(bn(y)).  With s = gamma * invstd, t = beta_bn - mean * s:
            //   dy = s * ([s y + t > 0] d - s1/N - xhat s2/N) = [s y + t > 0] * s * d + alpha * y + beta
            //   alpha = -s * invstd * s2 / N,  beta = -s * s1 / N - alpha * mean        (host: coda_bn_bwd_coefs)
            const float2 d = *reinterpret_cast<const float2 *>(rt + RAW_TILE + off);
            const float2 s2 = __ldg(reinterpret_cast<const float2 *>(P.scale + kc));
            const float2 h2 = __ldg(reinterpret_cast<const float2 *>(P.shift + kc));
            const float2 a2 = __ldg(reinterpret_cast<const float2 *>(P.alpha + kc));
            const float2 b2 = __ldg(reinterpret_cast<const float2 *>(P.beta + kc));
            x.x = (fmaf(x.x, s2.x, h2.x) > 0.f ? s2.x * d.x : 0.f) + fmaf(x.x, a2.x, b2.x);
            x.y = (fmaf(x.y, s2.y, h2.y) > 0.f ? s2.y * d.y : 0.f) + fmaf(x.y, a2.y, b2.y);
          } else if (P.mode == CODA_A32_BN_BWD_POOLED_PRE) {
            // pre-masked, pre-scaled pooled gradient: one compare + select + FMA + add per element
            const unsigned char *px = rt + RAW_TILE + pgt * 320;
            const float2 a2 = __ldg(reinterpret_cast<const float2 *>(P.alpha + kc));
            const float2 b2 = __ldg(reinterpret_cast<const float2 *>(P.beta + kc));
            const float2 d = *reinterpret_cast<const float2 *>(px + col * 4);
            const uchar2 id = *reinterpret_cast<const uchar2 *>(px + 256 + col);
            const int gi = pgi[q & 1];
            x.x = (id.x == gi ? d.x : 0.f) + fmaf(x.x, a2.x, b2.x);
            x.y = (id.y == gi ? d.y : 0.f) + fmaf(x.y, a2.y, b2.y);
          } else if (P.mode == CODA_A32_BN_BWD_POOLED) {
            // the layer output was max-pooled over `group` rows: only the arg-max row of a (group, channel)
            // carries the incoming gradient dpooled[g][c]
            const unsigned char *px = rt + RAW_TILE + pgt * 320;     // staged by the producer with the raw tile
            const float2 s2 = __ldg(reinterpret_cast<const float2 *>(P.scale + kc));
            const float2 h2 = __ldg(reinterpret_cast<const float2 *>(P.shift + kc));
            const float2 a2 = __ldg(reinterpret_cast<const float2 *>(P.alpha + kc));
            const float2 b2 = __ldg(reinterpret_cast<const float2 *>(P.beta + kc));
            const float2 d = *reinterpret_cast<const float2 *>(px + col * 4);
            const uchar2 id = *reinterpret_cast<const uchar2 *>(px + 256 + col);
            const int gi = pgi[q & 1];
            x.x = ((id.x == gi && fmaf(x.x, s2.x, h2.x) > 0.f) ? s2.x * d.x : 0.f) + fmaf(x.x, a2.x, b2.x);
            x.y = ((id.y == gi && fmaf(x.y, s2.y, h2.y) > 0.f) ? s2.y * d.y : 0.f) + fmaf(x.y, a2.y, b2.y);
          }
          uint32_t w[NSPLIT];
          split_pair<NSPLIT>(x.x, x.y, w);
#pragma unroll
          for (int pl = 0; pl < NSPLIT; ++pl) af[kk][pl][q] = w[pl];
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&raw_empty[rs]);    // this warp's rows of the raw stage have been read
      mbar_wait(&b_full[bs], P.b_resident ? 0u : ((it / B_STAGES) & 1u));
      unsigned char *bt = b_ring + (size_t)bs * B_STAGE;
      acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < n_products(NSPLIT); ++p) {
        const void *btile = bt + prod_b(NSPLIT, p) * B_TILE;
        const uint64_t bd = B_MN ? gmma_desc_mn_sw128(btile) : gmma_desc_k_sw128(btile);
        constexpr uint32_t KSTEP = B_MN ? 16 * 128 : 32;
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk)
          Wgmma<BN, false>::template rs<B_MN ? 1 : 0>(acc, af[kk][prod_a(NSPLIT, p)], gmma_desc_advance(bd, kk * KSTEP),
                                                      (kb | p | kk) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();     // the A fragments are overwritten by the next k-block
      acc_fence(acc);
      if (!P.b_resident && (threadIdx.x & 127) == 0) mbar_arrive(&b_empty[bs]);
    }

    // ===== epilogue: registers -> (+bias, ReLU) -> global, optional column statistics =====
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      const int col = n0 + c * 8 + 2 * t4;
      float cs0 = 0.f, cs1 = 0.f, cq0 = 0.f, cq1 = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = m0 + rloc[i];
        float v0 = acc[c * 4 + i * 2], v1 = acc[c * 4 + i * 2 + 1];
        if (P.bias) {
          if (col < n) v0 += __ldg(P.bias + col);
          if (col + 1 < n) v1 += __ldg(P.bias + col + 1);
        }
        if (P.act == 1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        if (row < m) {      // rows past m are padding: not stored, excluded from the statistics
          float *crow = P.c + (size_t)row * P.ldc;
          if (col + 1 < n) {
            *reinterpret_cast<float2 *>(crow + col) = make_float2(v0, v1);   // ldc % 4 == 0, col even
          } else if (col < n) {
            crow[col] = v0;
          }
          cs0 += v0; cq0 = fmaf(v0, v0, cq0);
          cs1 += v1; cq1 = fmaf(v1, v1, cq1);
        }
      }
      if (my_stats) {
        // column sums over the warp's 16 rows: reduce across the eight row groups (lane bits 2..4)
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
          cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
          cq0 += __shfl_xor_sync(0xffffffffu, cq0, o);
          cq1 += __shfl_xor_sync(0xffffffffu, cq1, o);
        }
        if (g == 0) {
          if (col < n) { my_stats[col] += cs0; my_stats[n + col] += cq0; }
          if (col + 1 < n) { my_stats[col + 1] += cs1; my_stats[n + col + 1] += cq1; }
        }
      }
    }
  }
  if (P.stats) {
    // fixed-order sum of the eight consumer warps' slices -> this CTA's partial row
    bar_sync(1, 256);
    float *out = P.stats + (size_t)blockIdx.x * 2 * n;
    for (int i = threadIdx.x; i < 2 * n; i += 256) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += s_stats[(size_t)w * 2 * n + i];
      out[i] = v;
    }
  }
}

int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int NSPLIT, int BN, int RAW_KB, int B_STAGES, bool B_MN>
int launch_a32(const A32Maps &maps, const A32Params &P, cudaStream_t s) {
  static_assert(RAW_KB % 64 == 0 || RAW_KB == 96, "raw region");
  constexpr size_t smem = (size_t)RAW_KB * 1024 + (size_t)B_STAGES * NSPLIT * BN * BK * 2 + 1024;
  const size_t total = smem + (P.stats ? (size_t)16 * P.n * 4 : 0);
  constexpr size_t SMEM_MAX = 227 * 1024 - 2048;     // static shared memory (barriers) shares the 227 KB limit
  if (total > SMEM_MAX) return CODA_ETOOLARGE;
  if (P.mode == CODA_A32_BN_BWD && RAW_KB < 64) return CODA_EINVAL;
  auto kern = gemm_a32_kernel<NSPLIT, BN, RAW_KB, B_STAGES, B_MN>;
  static size_t configured = 0;
  if (configured < total) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
    if (e != cudaSuccess) return (int)e;
    configured = SMEM_MAX;
  }
  const int tiles_m = (P.m + BM - 1) / BM, tiles_n = (P.n + BN - 1) / BN;
  const long long nwork = (long long)tiles_m * tiles_n;
  unsigned grid = (unsigned)(nwork < num_sms() ? nwork : num_sms());
  A32Params Q = P;
  const int nkb = (P.k + BK - 1) / BK;
  // short contraction, many m-tiles: keep the weights of one n-tile resident per CTA
  Q.b_resident = (nkb <= B_STAGES && tiles_n <= num_sms() && tiles_m >= 4 * (num_sms() / tiles_n)) ? 1 : 0;
  if (Q.b_resident) grid = (unsigned)((num_sms() / tiles_n) * tiles_n);
  kern<<<grid, A32_THREADS, total, s>>>(maps, Q);
  return launch_status();
}

}  // namespace

extern "C" {

int coda_gemm_a32_grid(int m, int n) {
  // upper bound of the launch grid = rows of the (zero-initialised) col_stats buffer the caller provides
  if (m <= 0 || n <= 0) return 0;
  return num_sms();
}

int coda_gemm_a32(int nsplit, int m, int n, int k, const float *a, long long lda, int a_mode, const float *a_scale,
                  const float *a_shift, const float *a_alpha, const float *a_beta, const float *a2, long long lda2,
                  const unsigned char *a_argmax, int a_group, const void *b_planes, long long b_plane_stride,
                  int b_ld, int b_mn, const float *bias, int act, float *c, long long ldc, float *col_stats,
                  void *stream) {
  if (nsplit < 2 || nsplit > 3 || m < 0 || n < 0 || k <= 0) return CODA_EINVAL;
  if (m == 0 || n == 0) return CODA_OK;
  if (!a || !b_planes || !c || b_ld % 64 != 0 || (lda & 3) || (ldc & 3) || ((uintptr_t)a & 15) || ((uintptr_t)c & 15))
    return CODA_EINVAL;
  if (a_mode < CODA_A32_PLAIN || a_mode > CODA_A32_BN_BWD_POOLED_PRE) return CODA_EINVAL;
  if (a_mode != CODA_A32_PLAIN && (!a_scale || !a_shift || (k & 3))) return CODA_EINVAL;
  if (a_mode >= CODA_A32_BN_BWD && (!a2 || !a_alpha || !a_beta || ((uintptr_t)a2 & 15))) return CODA_EINVAL;
  if (a_mode == CODA_A32_BN_BWD && (lda2 & 3)) return CODA_EINVAL;
  if ((a_mode == CODA_A32_BN_BWD_POOLED || a_mode == CODA_A32_BN_BWD_POOLED_PRE) &&
      (!a_argmax || a_group < 32 || a_group > 256 || m % a_group != 0 || k % 64 != 0 ||
       !(a_group % 128 == 0 || 128 % a_group == 0) || a_group % 32 != 0))
    return CODA_EINVAL;     // groups must tile the 128-row blocks (warp = 32 rows of one group)
  // few output tiles (the decoder's 2048-row linears: 16 x 4 tiles of 128 x 128 on 132 SMs): 64-wide tiles double
  // the number of CTAs at work; each of these launches is bounded by one CTA's serial tile time, not by throughput
  const long long tiles128 = (long long)((m + BM - 1) / BM) * ((n + 127) / 128);
  const int bn = (n <= 64 || tiles128 <= num_sms() / 2) ? 64 : 128;
  A32Maps maps;
  int st = make_tmap_f32_box(&maps.a, a, k, m, lda, 32, BM);
  if (st != CODA_OK) return st;
  maps.a2 = maps.a;
  if (a_mode == CODA_A32_BN_BWD) {
    st = make_tmap_f32_box(&maps.a2, a2, k, m, lda2, 32, BM);
    if (st != CODA_OK) return st;
  }
  const int kpad = (k + 63) / 64 * 64;
  const char *bp = (const char *)b_planes;
  for (int p = 0; p < nsplit; ++p) {
    if (!b_mn) {
      // planes [n rows][b_ld >= kpad], K contiguous; box [bn rows][64]
      if (b_ld < kpad) return CODA_EINVAL;
      st = make_tmap_k_major_16b(&maps.b[p], bp + (size_t)p * b_plane_stride * 2, 0, b_ld, n, 1, b_ld, 0, bn);
    } else {
      // planes [k rows][b_ld >= n], N contiguous (the forward weight planes, used for dX = dY W); box [64][64]
      if (b_ld < n) return CODA_EINVAL;
      st = make_tmap_k_major_16b(&maps.b[p], bp + (size_t)p * b_plane_stride * 2, 0, b_ld, k, 1, b_ld, 0, 64);
    }
    if (st != CODA_OK) return st;
  }
  for (int p = nsplit; p < 3; ++p) maps.b[p] = maps.b[0];
  A32Params P;
  P.m = m; P.n = n; P.k = k; P.mode = a_mode; P.scale = a_scale; P.shift = a_shift; P.alpha = a_alpha; P.beta = a_beta;
  P.dpooled = a2; P.argmax = a_argmax; P.group = a_group; P.bias = bias; P.act = act; P.c = c; P.ldc = ldc; P.stats = col_stats;
  P.b_resident = 0;
  cudaStream_t s = (cudaStream_t)stream;
#define CODA_A32(NS, BN_, RS, BS)                                                   \
  return b_mn ? launch_a32<NS, BN_, RS, BS, true>(maps, P, s) : launch_a32<NS, BN_, RS, BS, false>(maps, P, s)
  // smem: raw region + B ring (+ stats): <= 225 KB.  The B (weight) tiles come from L2 with ~1 us
  // latency: long contractions want a deep B ring, the two-input prologue a wide raw region.
  const bool deep_b = !col_stats && k > 128 && a_mode != CODA_A32_BN_BWD;
  if (nsplit == 2) {
    if (bn == 64) CODA_A32(2, 64, 128, 4);
    CODA_A32(2, 128, 128, 2);
  }
  if (bn == 64) CODA_A32(3, 64, 128, 3);
  if (deep_b) CODA_A32(3, 128, 64, 3);
  CODA_A32(3, 128, 96, 2);
#undef CODA_A32
}

}  // extern "C"
