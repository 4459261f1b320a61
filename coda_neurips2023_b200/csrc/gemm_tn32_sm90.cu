// Weight-gradient GEMM on fp32 ROWS with in-kernel prologues (wgmma, sm_90a):
//
//     C[m][n] = sum_r  TA(A)[r][m] * TB(B)[r][n]          (dW = dY^T X, contraction over the ROWS of both operands)
//
// A (R, M) and B (R, N) are the row-major fp32 activations as they sit in HBM.  In gemm_sm90.cu's TN form both have
// to exist as row-packed bf16 planes first (a pack kernel per operand: read 4 B, write 4 B, read 4 B again per
// element); here every 32-row slab is TMA-loaded as fp32, the consumer warps apply the prologue
//     TA: identity | BatchNorm+ReLU backward of the layer (dense two-input form, or max-pooled form)
//     TB: identity | BatchNorm+ReLU forward of the previous layer (relu(b * scale + shift))
// split the values into two bf16 planes and write them as MN-major, 128B-swizzled wgmma operands in shared
// memory.  The kernel is a pure stream over R: split-K across all SMs; every split stores its partial tile in a
// scratch slot and tn32_splitk_reduce_kernel adds the slots in split order (the same result on every run).
//
// Warp roles (288 threads): 8 TMA producer | 0-7 transform (four rows of each operand slab per warp), then the same
// warps as two wgmma warpgroups (rows [0, 64) and [64, 128) of the tile) on the converted slab.  Three converted slabs
// are in flight, so the transform of slab i overlaps the MMAs of slab i-1.
// The launch streams from HBM, so the raw ring is as deep as shared memory allows: a raw stage holds only what the A
// prologue mode reads (the second A input only in the dense BatchNorm-backward mode, the pooled gradient row only in
// the max-pooled modes), the stage count is fixed per (BN, mode) at compile time, and a warp frees its share of a stage
// as soon as its rows are in registers, before the split and the plane stores.
// Optional: the column sums of TA(A) (the bias gradient of the layer whose dW this is) are accumulated by the
// transform warps on the way -- the values are in registers already -- instead of a separate pass over dY.
// C-ABI in include/coda_gemm.h (coda_gemm_tn32).
#include "../../include/coda_gemm.h"
#include "a32_prologue.cuh"
#include "sm90_primitives.cuh"

using namespace coda;

namespace {

constexpr int BM = 128;      // output rows per tile  (columns of A)
constexpr int BKR = 32;      // contraction rows per pipeline stage
constexpr int NS = 2;        // bf16 planes per operand (gradient precision, as the packed TN path)
constexpr int PL_STAGES = 3;  // converted operand slabs (slab i's planes are rewritten after the MMAs of i - 1 retire)
constexpr int TW = 8;        // transform warps (= the two consumer warpgroups)
constexpr int TN32_THREADS = 288;

// What a raw stage carries, by A prologue mode: the A slab and the B slab always, the second A input of the dense
// BatchNorm-backward mode, or the slab's pooled-gradient row and arg-max bytes in the max-pooled modes.
enum RawKind { RAW_PLAIN = 0, RAW_POOLED = 1, RAW_DENSE = 2 };

__host__ inline int raw_kind(int a_mode) {
  if (a_mode == CODA_A32_BN_BWD) return RAW_DENSE;
  if (a_mode == CODA_A32_BN_BWD_POOLED || a_mode == CODA_A32_BN_BWD_POOLED_PRE) return RAW_POOLED;
  return RAW_PLAIN;
}

// Shared-memory layout of one (BN, kind) instance: RAW_STAGES fp32 stages [A | A2 (dense) | B | pooled row (pooled)],
// then PL_STAGES bf16 plane stages.  The raw ring takes what the plane ring and the static arrays leave of the 227 KB.
template <int BN, int KIND>
struct TN32Layout {
  static constexpr int RAW_A = BKR * BM * 4;     // 16 KB: four [32 rows x 32 fp32] SW128 boxes
  static constexpr int RAW_B = BKR * BN * 4;
  static constexpr int OFF_B = KIND == RAW_DENSE ? 2 * RAW_A : RAW_A;
  static constexpr int OFF_X = OFF_B + RAW_B;    // pooled: [128 floats dpooled | 128 bytes argmax] of the slab's group
  static constexpr int RAW_STAGE = OFF_X + (KIND == RAW_POOLED ? 1024 : 0);   // 1024-aligned: the boxes are SW128
  static constexpr int PL_A = BKR * BM * 2;      // one bf16 plane of the A slab: two [32 x 64] boxes
  static constexpr int PL_B = BKR * BN * 2;
  static constexpr int PL_STAGE = NS * (PL_A + PL_B);
  // 227 KB less the 1 KB alignment slack and the static arrays (column sums and mbarriers, padded to 1 KB: 5 KB)
  static constexpr int BUDGET = 227 * 1024 - 1024 - (TW * BM * 4 + 1024);
  static constexpr int RAW_STAGES_FIT = (BUDGET - PL_STAGES * PL_STAGE) / RAW_STAGE;
  // The dense mode keeps two stages (40 / 48 KB each): a third made SA layer 2's weight gradient, which streams at
  // ~90 % of HBM with two, slower.
  static constexpr int RAW_STAGES = KIND == RAW_DENSE ? 2 : (RAW_STAGES_FIT < 6 ? RAW_STAGES_FIT : 6);
  static constexpr size_t SMEM = (size_t)RAW_STAGES * RAW_STAGE + (size_t)PL_STAGES * PL_STAGE + 1024;
  static_assert(RAW_STAGES >= 2, "raw ring");
};

struct TN32Maps {
  CUtensorMap a, a2, b;
};

struct TN32Params {
  long long rows;
  int m, n;
  int a_mode, b_mode;        // CODA_A32_*
  const float *a_scale, *a_shift, *a_alpha, *a_beta;    // per column of A (padded to a multiple of 128)
  const float *dpooled;      // pooled form: (rows / group, m)
  const unsigned char *argmax;
  int group;
  const float *b_scale, *b_shift;                       // per column of B (padded)
  float *a_colsum;           // optional (m): column sums of TA(A)
  float *partial;            // split-K scratch: [tiles][ksplit][BM][BN] partial tiles, then [tiles_m][ksplit][BM] column sums
  float *c;
  long long ldc;
  int ksplit;
};

template <int BN, int KIND>
__global__ void __launch_bounds__(TN32_THREADS, 1)
gemm_tn32_kernel(const __grid_constant__ TN32Maps maps, const TN32Params P) {
  using L = TN32Layout<BN, KIND>;
  constexpr int RAW_A = L::RAW_A, OFF_B = L::OFF_B, OFF_X = L::OFF_X;
  constexpr int RAW_STAGE = L::RAW_STAGE, RAW_STAGES = L::RAW_STAGES;
  constexpr int PL_A = L::PL_A, PL_B = L::PL_B, PL_STAGE = L::PL_STAGE;
  constexpr bool two_in = KIND == RAW_DENSE, pooled_mode = KIND == RAW_POOLED;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // rounded up to 1024 bytes by an offset from the shared array itself (not through an integer address), so that the
  // compiler keeps the shared address space: LDS / STS in the transform, not generic loads and stores
  unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char *raw_ring = smem;
  unsigned char *pl_ring = smem + (size_t)RAW_STAGES * RAW_STAGE;
  __shared__ __align__(8) uint64_t raw_full[RAW_STAGES], raw_empty[RAW_STAGES];
  __shared__ __align__(16) float s_colsum[TW][BM];   // per-warp column sums of TA(A), added in warp order

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_n = (P.n + BN - 1) / BN;
  const int tile = blockIdx.x / P.ksplit, ks = blockIdx.x % P.ksplit;
  const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
  const long long nkb_total = (P.rows + BKR - 1) / BKR;
  const long long per = (nkb_total + P.ksplit - 1) / P.ksplit;
  const long long kb0 = (long long)ks * per;
  const long long nkb = max(0ll, min(per, nkb_total - kb0));

  if (threadIdx.x == 0) {
    for (int s = 0; s < RAW_STAGES; ++s) { mbar_init(&raw_full[s], 1); mbar_init(&raw_empty[s], TW); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      prefetch_tmap(&maps.a);
      prefetch_tmap(&maps.b);
      if (two_in) prefetch_tmap(&maps.a2);
    }
    constexpr uint32_t bytes = (uint32_t)(OFF_X + (pooled_mode ? 640 : 0));
    const long long ngroups = pooled_mode ? P.rows / P.group : 0;
    for (long long i = 0; i < nkb; ++i) {
      const int rs = (int)(i % RAW_STAGES);
      mbar_wait(&raw_empty[rs], (uint32_t)((i / RAW_STAGES) & 1) ^ 1u);
      if (elect_one_sync()) {
        unsigned char *st = raw_ring + (size_t)rs * RAW_STAGE;
        const int r0 = (int)((kb0 + i) * BKR);
        mbar_arrive_expect_tx(&raw_full[rs], bytes);
        if constexpr (pooled_mode) {      // the slab (32 rows) lies in one group (group % 32 == 0)
          long long g = (long long)r0 / P.group;
          if (g >= ngroups) g = ngroups - 1;
          // m0 + 128 <= padded m: the host guarantees m % 128 == 0 in this mode
          bulk_load_1d(st + OFF_X, P.dpooled + g * P.m + m0, 512, &raw_full[rs]);
          bulk_load_1d(st + OFF_X + 512, P.argmax + g * P.m + m0, 128, &raw_full[rs]);
        }
#pragma unroll
        for (int g = 0; g < BM / 32; ++g) tma_load_3d(st + g * 4096, &maps.a, &raw_full[rs], m0 + g * 32, r0, 0);
        if constexpr (two_in) {
#pragma unroll
          for (int g = 0; g < BM / 32; ++g) tma_load_3d(st + RAW_A + g * 4096, &maps.a2, &raw_full[rs], m0 + g * 32, r0, 0);
        }
#pragma unroll
        for (int g = 0; g < BN / 32; ++g) tma_load_3d(st + OFF_B + g * 4096, &maps.b, &raw_full[rs], n0 + g * 32, r0, 0);
      }
      __syncwarp();
    }
    return;
  }

  // ===== transform: fp32 slabs -> prologue -> two bf16 planes, MN-major swizzled; then wgmma on them =====
  const int tw = warp;                             // rows tw, tw + 8, tw + 16, tw + 24 of the slab
  const int wg = warp >> 2;
  const bool want_colsum = P.a_colsum != nullptr && n0 == 0;
  float4 csum = make_float4(0.f, 0.f, 0.f, 0.f);
  // A: lane = 4-column chunk (128 columns = 32 chunks);  per-column coefficients live in registers
  const int ca = m0 + lane * 4;
  float4 sa = make_float4(0.f, 0.f, 0.f, 0.f), ta = sa, al = sa, be = sa;
  if (P.a_mode != CODA_A32_PLAIN && ca < P.m) {
    sa = __ldg(reinterpret_cast<const float4 *>(P.a_scale + ca));
    ta = __ldg(reinterpret_cast<const float4 *>(P.a_shift + ca));
    al = __ldg(reinterpret_cast<const float4 *>(P.a_alpha + ca));
    be = __ldg(reinterpret_cast<const float4 *>(P.a_beta + ca));
  }
  // B: BN / 4 chunks per row; with BN = 64 a warp covers two rows per pass
  constexpr int B_CHUNKS = BN / 4, B_RPP = 32 / B_CHUNKS;        // rows per pass
  const int bch = lane % B_CHUNKS, brow_off = lane / B_CHUNKS;
  const int cb = n0 + bch * 4;
  float4 sb = make_float4(0.f, 0.f, 0.f, 0.f), tb = sb;
  if (P.b_mode == CODA_A32_AFFINE_RELU && cb < P.n) {
    sb = __ldg(reinterpret_cast<const float4 *>(P.b_scale + cb));
    tb = __ldg(reinterpret_cast<const float4 *>(P.b_shift + cb));
  }
  // the slab's first row within its group, carried from slab to slab (group >= 32 = BKR: one conditional subtract)
  int rem0 = pooled_mode ? (int)((kb0 * BKR) % P.group) : 0;
  int rs = 0, ps = 0;
  uint32_t raw_par = 0;
  float acc[BN / 2];
  for (long long i = 0; i < nkb; ++i) {
    // plane stage ps last held slab i - 3, whose MMAs every warpgroup had waited for before the barrier of slab i - 1
    mbar_wait_relaxed(&raw_full[rs], raw_par);
    const unsigned char *raw = raw_ring + (size_t)rs * RAW_STAGE;
    unsigned char *pl = pl_ring + (size_t)ps * PL_STAGE;
    const long long r0 = (kb0 + i) * BKR;
    const bool tail = r0 + BKR > P.rows;
      // ---- the warp's rows of both slabs, prologues applied, into registers; then its share of the raw stage is free
      float4 oa[BKR / TW], ob[BKR / (TW * B_RPP)];
      float4 dp = make_float4(0.f, 0.f, 0.f, 0.f);
      uchar4 id = make_uchar4(0, 0, 0, 0);
      if constexpr (pooled_mode) {   // the slab's pooled-gradient row and arg-max bytes: one group, the same for every row
        dp = *reinterpret_cast<const float4 *>(raw + OFF_X + lane * 16);
        id = *reinterpret_cast<const uchar4 *>(raw + OFF_X + 512 + lane * 4);
      }
#pragma unroll
      for (int j = 0; j < BKR / (TW * B_RPP); ++j) {
        const int r = (tw + j * TW) * B_RPP + brow_off;
        const uint32_t roff = (uint32_t)(bch >> 3) * 4096u + (uint32_t)r * 128u + (uint32_t)(((bch & 7) ^ (r & 7)) << 4);
        float4 v = *reinterpret_cast<const float4 *>(raw + OFF_B + roff);
        if (P.b_mode == CODA_A32_AFFINE_RELU) {
          v.x = a32::affine_relu(v.x, sb.x, tb.x); v.y = a32::affine_relu(v.y, sb.y, tb.y);
          v.z = a32::affine_relu(v.z, sb.z, tb.z); v.w = a32::affine_relu(v.w, sb.w, tb.w);
        }
        ob[j] = v;
      }
      if (tail) {                    // only the very last slab can hold rows past the end: zero its padding rows
#pragma unroll
        for (int j = 0; j < BKR / (TW * B_RPP); ++j)
          if (r0 + (tw + j * TW) * B_RPP + brow_off >= P.rows) ob[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      const auto store_b = [&] {
#pragma unroll
        for (int j = 0; j < BKR / (TW * B_RPP); ++j) {
          const int r = (tw + j * TW) * B_RPP + brow_off, col = bch * 4;
          split_store4<NS>(ob[j], reinterpret_cast<__nv_bfloat16 *>(pl + NS * PL_A + (col >> 6) * (BKR * 128) + r * 128 +
                                                                    ((((col & 63) >> 3) ^ (r & 7)) << 4) + ((col & 7) >> 2) * 8),
                           PL_B / 2);
        }
      };
      if constexpr (two_in) store_b();    // holding the B rows while both A inputs are read spilled at BN = 128
#pragma unroll
      for (int j = 0; j < BKR / TW; ++j) {
        const int r = tw + j * TW;
        const uint32_t roff = (uint32_t)(lane >> 3) * 4096u + (uint32_t)r * 128u + (uint32_t)(((lane & 7) ^ (r & 7)) << 4);
        float4 y = *reinterpret_cast<const float4 *>(raw + roff);
        float4 o = y;
        if constexpr (two_in) {
          const float4 d = *reinterpret_cast<const float4 *>(raw + RAW_A + roff);
          o.x = a32::bn_bwd(y.x, d.x, sa.x, ta.x, al.x, be.x);
          o.y = a32::bn_bwd(y.y, d.y, sa.y, ta.y, al.y, be.y);
          o.z = a32::bn_bwd(y.z, d.z, sa.z, ta.z, al.z, be.z);
          o.w = a32::bn_bwd(y.w, d.w, sa.w, ta.w, al.w, be.w);
        } else if constexpr (pooled_mode) {
          const int gi = rem0 + r;
          if (P.a_mode == CODA_A32_BN_BWD_POOLED_PRE) {
            o.x = a32::bn_bwd_pooled_pre(y.x, dp.x, id.x == gi, al.x, be.x);
            o.y = a32::bn_bwd_pooled_pre(y.y, dp.y, id.y == gi, al.y, be.y);
            o.z = a32::bn_bwd_pooled_pre(y.z, dp.z, id.z == gi, al.z, be.z);
            o.w = a32::bn_bwd_pooled_pre(y.w, dp.w, id.w == gi, al.w, be.w);
          } else {
            o.x = a32::bn_bwd_pooled(y.x, dp.x, id.x == gi, sa.x, ta.x, al.x, be.x);
            o.y = a32::bn_bwd_pooled(y.y, dp.y, id.y == gi, sa.y, ta.y, al.y, be.y);
            o.z = a32::bn_bwd_pooled(y.z, dp.z, id.z == gi, sa.z, ta.z, al.z, be.z);
            o.w = a32::bn_bwd_pooled(y.w, dp.w, id.w == gi, sa.w, ta.w, al.w, be.w);
          }
        }
        oa[j] = o;
      }
      if (tail) {
#pragma unroll
        for (int j = 0; j < BKR / TW; ++j)
          if (r0 + tw + j * TW >= P.rows) oa[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (want_colsum) {
#pragma unroll
        for (int j = 0; j < BKR / TW; ++j) { csum.x += oa[j].x; csum.y += oa[j].y; csum.z += oa[j].z; csum.w += oa[j].w; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&raw_empty[rs]);    // the producer may refill the stage while the planes are written
      // ---- two bf16 planes of each operand, MN-major swizzled
      // destination: box = column / 64, 16-byte chunk = (column % 64) / 8 swizzled by the row, half = (column % 8) / 4
#pragma unroll
      for (int j = 0; j < BKR / TW; ++j) {
        const int r = tw + j * TW, col = lane * 4;
        split_store4<NS>(oa[j], reinterpret_cast<__nv_bfloat16 *>(pl + (col >> 6) * (BKR * 128) + r * 128 +
                                                                  ((((col & 63) >> 3) ^ (r & 7)) << 4) + ((col & 7) >> 2) * 8),
                         PL_A / 2);
      }
      if constexpr (!two_in) store_b();
      fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core's async-proxy reads
      bar_sync(1, 256);              // both operand slabs are complete in shared memory
      // plane products; the warpgroup's 64 rows are the A slab's box wg
      acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < n_products(NS); ++p) {
        const uint64_t ad = gmma_desc_mn_sw128(pl + prod_a(NS, p) * PL_A + wg * (BKR * 128), BKR * 128);
        const uint64_t bd = gmma_desc_mn_sw128(pl + NS * PL_A + prod_b(NS, p) * PL_B, BKR * 128);
#pragma unroll
        for (int kk = 0; kk < BKR / 16; ++kk)
          Wgmma<BN, false>::template ss<1, 1>(acc, gmma_desc_advance(ad, kk * 16 * 128), gmma_desc_advance(bd, kk * 16 * 128),
                                              (i | p | kk) != 0);
      }
      wgmma_commit();
      wgmma_wait<1>();
      acc_fence(acc);
      if (++rs == RAW_STAGES) { rs = 0; raw_par ^= 1u; }
      if (++ps == PL_STAGES) ps = 0;
      if (pooled_mode) { rem0 += BKR; if (rem0 >= P.group) rem0 -= P.group; }
  }
  wgmma_wait<0>();
  acc_fence(acc);
  if (nkb == 0) acc_zero(acc);     // a split past the last slab contributes zeros
  *reinterpret_cast<float4 *>(&s_colsum[tw][lane * 4]) = csum;
  // ===== epilogue: registers -> C, or (split-K) -> the split's scratch slot, added in split order by tn32_splitk_reduce_kernel

  {
    const int g = lane >> 2, t4 = lane & 3;
    float *slot = P.partial + ((long long)tile * P.ksplit + ks) * (BM * BN);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int rl = wg * 64 + (warp & 3) * 16 + g + 8 * i, row = m0 + rl;
      float *crow = P.c + (size_t)row * P.ldc;
#pragma unroll
      for (int c = 0; c < BN / 8; ++c) {
        const int col = n0 + c * 8 + 2 * t4;
        const float2 v = make_float2(acc[c * 4 + i * 2], acc[c * 4 + i * 2 + 1]);
        if (P.ksplit > 1) *reinterpret_cast<float2 *>(slot + (size_t)rl * BN + c * 8 + 2 * t4) = v;
        else if (row < P.m && col < P.n) *reinterpret_cast<float2 *>(crow + col) = v;   // n % 4 == 0: col + 1 < n
      }
    }
  }
  bar_sync(1, 256);
  if (P.a_colsum && n0 == 0 && threadIdx.x < BM) {
    float cs = 0.f;
#pragma unroll
    for (int w = 0; w < TW; ++w) cs += s_colsum[w][threadIdx.x];
    if (P.ksplit > 1) {
      const int tiles_m = (P.m + BM - 1) / BM;
      P.partial[(long long)tiles_m * (tiles_n * P.ksplit) * (BM * BN) + ((long long)(m0 / BM) * P.ksplit + ks) * BM +
                threadIdx.x] = cs;
    } else if (m0 + (int)threadIdx.x < P.m) {
      P.a_colsum[m0 + threadIdx.x] = cs;
    }
  }
}

// C of the split-K launch: the scratch slots of a tile added in split order, as splitk_reduce_kernel adds them
// (0 + slot 0 + slot 1 + ...: the same bits).  A thread owns four columns of one tile row: float4 loads and stores and
// 32-bit index arithmetic instead of one column per thread and 64-bit divisions.  n % 4 == 0, ldc % 4 == 0 and a
// 16-byte aligned C are checked by coda_gemm_tn32.
template <int BN>
__global__ void __launch_bounds__(256)
tn32_splitk_reduce_kernel(const float *__restrict__ partial, int ksplit, int m, int n, float *__restrict__ c,
                          long long ldc) {
  constexpr int QUADS = BN / 4;
  const int tiles_n = (n + BN - 1) / BN, tiles = ((m + BM - 1) / BM) * tiles_n;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int tile = idx / (BM * QUADS), rl = (idx / QUADS) % BM, q = idx % QUADS;
  if (tile >= tiles) return;
  const int row = (tile / tiles_n) * BM + rl, col = (tile % tiles_n) * BN + q * 4;
  if (row >= m || col >= n) return;
  const float4 *src = reinterpret_cast<const float4 *>(partial + (size_t)tile * ksplit * (BM * BN) + rl * BN) + q;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = 0; k < ksplit; ++k) {
    const float4 p = __ldg(src + (size_t)k * (BM * BN / 4));
    v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
  }
  *reinterpret_cast<float4 *>(c + (size_t)row * ldc + col) = v;
}

// column sums of the split-K launch: a_colsum[col] = sum_k parts[(col / BM) * ksplit + k][col % BM], in split order
__global__ void __launch_bounds__(256)
colsum_reduce_kernel(const float *__restrict__ parts, int ksplit, int m, float *__restrict__ a_colsum) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= m) return;
  const float *src = parts + ((long long)(col / BM) * ksplit) * BM + col % BM;
  float v = 0.f;
  for (int k = 0; k < ksplit; ++k) v += src[(long long)k * BM];
  a_colsum[col] = v;
}

// the kernel instance of one raw-stage kind, with its shared-memory limit raised
template <int BN, int KIND>
int tn32_instance(void (**kern)(TN32Maps, TN32Params), size_t *smem) {
  constexpr auto k = gemm_tn32_kernel<BN, KIND>;
  *kern = k;
  *smem = TN32Layout<BN, KIND>::SMEM;
  return raise_smem_limit<k>((int)*smem);
}

template <int BN>
int launch_tn32(const TN32Maps &maps, TN32Params P, float *c, long long ldc, cudaStream_t s) {
  void (*kern)(TN32Maps, TN32Params) = nullptr;
  size_t smem = 0;
  const int kind = raw_kind(P.a_mode);
  const int st0 = kind == RAW_DENSE    ? tn32_instance<BN, RAW_DENSE>(&kern, &smem)
                  : kind == RAW_POOLED ? tn32_instance<BN, RAW_POOLED>(&kern, &smem)
                                       : tn32_instance<BN, RAW_PLAIN>(&kern, &smem);
  if (st0 != CODA_OK) return st0;
  const int num_sms = sm_count();
  const int tiles = ((P.m + BM - 1) / BM) * ((P.n + BN - 1) / BN);
  const long long nkb_total = (P.rows + BKR - 1) / BKR;
  int ksplit = num_sms / tiles;
  if (ksplit < 1) ksplit = 1;
  if (ksplit > nkb_total / 4) ksplit = (int)(nkb_total / 4 > 0 ? nkb_total / 4 : 1);   // >= 4 slabs per CTA
  P.ksplit = ksplit;
  const int tiles_m = (P.m + BM - 1) / BM;
  if (ksplit > 1) {
    const int st = split_scratch((size_t)tiles * ksplit * BM * BN + (size_t)tiles_m * ksplit * BM, s, &P.partial);
    if (st != CODA_OK) return st;
  }
  kern<<<tiles * ksplit, TN32_THREADS, smem, s>>>(maps, P);
  if (ksplit > 1) {
    const int threads = tiles * BM * (BN / 4);
    tn32_splitk_reduce_kernel<BN><<<(threads + 255) / 256, 256, 0, s>>>(P.partial, ksplit, P.m, P.n, c, ldc);
    if (P.a_colsum)
      colsum_reduce_kernel<<<(P.m + 255) / 256, 256, 0, s>>>(P.partial + (size_t)tiles * ksplit * BM * BN, ksplit, P.m,
                                                            P.a_colsum);
  }
  return launch_status();
}

}  // namespace

extern "C" {

int coda_gemm_tn32(long long rows, int m, int n, const float *a, long long lda, int a_mode, const float *a_scale,
                   const float *a_shift, const float *a_alpha, const float *a_beta, const float *a2, long long lda2,
                   const unsigned char *a_argmax, int a_group, const float *b, long long ldb, int b_mode,
                   const float *b_scale, const float *b_shift, float *c, long long ldc, float *a_colsum, void *stream) {
  if (rows <= 0 || m <= 0 || n <= 0 || !a || !b || !c) return CODA_EINVAL;
  if ((lda & 3) || (ldb & 3) || (ldc & 3) || (m & 3) || (n & 3)) return CODA_EINVAL;
  if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15) return CODA_EINVAL;
  if (a_mode != CODA_A32_PLAIN && a_mode != CODA_A32_BN_BWD && a_mode != CODA_A32_BN_BWD_POOLED &&
      a_mode != CODA_A32_BN_BWD_POOLED_PRE)
    return CODA_EINVAL;
  if (b_mode != CODA_A32_PLAIN && b_mode != CODA_A32_AFFINE_RELU) return CODA_EINVAL;
  if (a_mode != CODA_A32_PLAIN && (!a_scale || !a_shift || !a_alpha || !a_beta || !a2 || ((uintptr_t)a2 & 15))) return CODA_EINVAL;
  if (a_mode == CODA_A32_BN_BWD && (lda2 & 3)) return CODA_EINVAL;
  if ((a_mode == CODA_A32_BN_BWD_POOLED || a_mode == CODA_A32_BN_BWD_POOLED_PRE) &&
      (!a_argmax || a_group < 32 || a_group > 256 || a_group % 32 != 0 || rows % a_group != 0 || m % 128 != 0))
    return CODA_EINVAL;     // a 32-row slab must lie in one group; the group rows are staged 128 columns at a time
  if (b_mode == CODA_A32_AFFINE_RELU && (!b_scale || !b_shift)) return CODA_EINVAL;
  TN32Maps maps;
  int st = make_tmap_f32_box(&maps.a, a, m, rows, lda, 32, BKR);
  if (st != CODA_OK) return st;
  maps.a2 = maps.a;
  if (a_mode == CODA_A32_BN_BWD) {
    st = make_tmap_f32_box(&maps.a2, a2, m, rows, lda2, 32, BKR);
    if (st != CODA_OK) return st;
  }
  st = make_tmap_f32_box(&maps.b, b, n, rows, ldb, 32, BKR);
  if (st != CODA_OK) return st;
  TN32Params P;
  P.rows = rows; P.m = m; P.n = n; P.a_mode = a_mode; P.b_mode = b_mode;
  P.a_scale = a_scale; P.a_shift = a_shift; P.a_alpha = a_alpha; P.a_beta = a_beta;
  P.dpooled = a2; P.argmax = a_argmax; P.group = a_group; P.b_scale = b_scale; P.b_shift = b_shift; P.a_colsum = a_colsum; P.partial = nullptr; P.c = c; P.ldc = ldc; P.ksplit = 1;
  cudaStream_t s = (cudaStream_t)stream;
  if (n <= 64) return launch_tn32<64>(maps, P, c, ldc, s);
  return launch_tn32<128>(maps, P, c, ldc, s);
}

}  // extern "C"
