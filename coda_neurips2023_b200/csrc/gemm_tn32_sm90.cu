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
// scratch slot and splitk_reduce_kernel adds the slots in split order (the same result on every run).
//
// Warp roles (288 threads): 8 TMA producer | 0-7 transform (four rows of each operand slab per warp), then the same
// warps as two wgmma warpgroups (rows [0, 64) and [64, 128) of the tile) on the converted slab.  Three converted slabs
// are in flight, so the transform of slab i overlaps the MMAs of slab i-1.
// Optional: the column sums of TA(A) (the bias gradient of the layer whose dW this is) are accumulated by the
// transform warps on the way -- the values are in registers already -- instead of a separate pass over dY.
// C-ABI in include/coda_gemm.h (coda_gemm_tn32).
#include "../../include/coda_gemm.h"
#include "sm90_primitives.cuh"

using namespace coda;

namespace {

constexpr int BM = 128;      // output rows per tile  (columns of A)
constexpr int BKR = 32;      // contraction rows per pipeline stage
constexpr int NS = 2;        // bf16 planes per operand (gradient precision, as the packed TN path)
constexpr int RAW_STAGES = 2, PL_STAGES = 3;   // fp32 slabs in flight (HBM latency) / converted operand slabs
constexpr int TW = 8;        // transform warps (= the two consumer warpgroups)
constexpr int TN32_THREADS = 288;

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

__device__ __forceinline__ void store_planes4(float4 v, unsigned char *dst, uint32_t plane_bytes) {
  float r[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int p = 0; p < NS; ++p) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(r[0], r[1]), hi = __floats2bfloat162_rn(r[2], r[3]);
    uint2 w;
    w.x = *reinterpret_cast<const uint32_t *>(&lo);
    w.y = *reinterpret_cast<const uint32_t *>(&hi);
    *reinterpret_cast<uint2 *>(dst + (size_t)p * plane_bytes) = w;
    if (p + 1 < NS) {
      r[0] -= __uint_as_float(w.x << 16); r[1] -= __uint_as_float(w.x & 0xFFFF0000u);
      r[2] -= __uint_as_float(w.y << 16); r[3] -= __uint_as_float(w.y & 0xFFFF0000u);
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(TN32_THREADS, 1)
gemm_tn32_kernel(const __grid_constant__ TN32Maps maps, const TN32Params P) {
  constexpr int RAW_A = BKR * BM * 4;            // 16 KB: four [32 rows x 32 fp32] SW128 boxes
  constexpr int RAW_B = BKR * BN * 4;
  constexpr int RAW_X = 1024;                    // pooled mode: [128 floats dpooled | 128 bytes argmax] of the slab's group
  constexpr int RAW_STAGE = 2 * RAW_A + RAW_B + RAW_X;   // (second A input only in the dense BN-backward mode)
  constexpr int PL_A = BKR * BM * 2;             // one bf16 plane of the A slab: two [32 x 64] boxes
  constexpr int PL_B = BKR * BN * 2;
  constexpr int PL_STAGE = NS * (PL_A + PL_B);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
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
  const bool two_in = P.a_mode == CODA_A32_BN_BWD;

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
    const bool pooled = P.a_mode == CODA_A32_BN_BWD_POOLED || P.a_mode == CODA_A32_BN_BWD_POOLED_PRE;
    const uint32_t bytes = (uint32_t)(RAW_A * (two_in ? 2 : 1) + RAW_B + (pooled ? 640 : 0));
    const long long ngroups = pooled ? P.rows / P.group : 0;
    for (long long i = 0; i < nkb; ++i) {
      const int rs = (int)(i % RAW_STAGES);
      mbar_wait(&raw_empty[rs], (uint32_t)((i / RAW_STAGES) & 1) ^ 1u);
      if (elect_one_sync()) {
        unsigned char *st = raw_ring + (size_t)rs * RAW_STAGE;
        const int r0 = (int)((kb0 + i) * BKR);
        mbar_arrive_expect_tx(&raw_full[rs], bytes);
        if (pooled) {      // the slab (32 rows) lies in one group (group % 32 == 0)
          long long g = (long long)r0 / P.group;
          if (g >= ngroups) g = ngroups - 1;
          // m0 + 128 <= padded m: the host guarantees m % 128 == 0 in this mode
          bulk_load_1d(st + 2 * RAW_A + RAW_B, P.dpooled + g * P.m + m0, 512, &raw_full[rs]);
          bulk_load_1d(st + 2 * RAW_A + RAW_B + 512, P.argmax + g * P.m + m0, 128, &raw_full[rs]);
        }
#pragma unroll
        for (int g = 0; g < BM / 32; ++g) tma_load_3d(st + g * 4096, &maps.a, &raw_full[rs], m0 + g * 32, r0, 0);
        if (two_in) {
#pragma unroll
          for (int g = 0; g < BM / 32; ++g) tma_load_3d(st + RAW_A + g * 4096, &maps.a2, &raw_full[rs], m0 + g * 32, r0, 0);
        }
#pragma unroll
        for (int g = 0; g < BN / 32; ++g) tma_load_3d(st + 2 * RAW_A + g * 4096, &maps.b, &raw_full[rs], n0 + g * 32, r0, 0);
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
  const bool a_col_ok = ca < P.m;
  const bool pooled_mode = P.a_mode == CODA_A32_BN_BWD_POOLED || P.a_mode == CODA_A32_BN_BWD_POOLED_PRE;
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
    const bool tail = r0 + BKR > P.rows;         // only the very last slab can hold rows past the end
      // ---- A slab
#pragma unroll
      for (int j = 0; j < BKR / TW; ++j) {
        const int r = tw + j * TW;
        const long long grow = r0 + r;
        const uint32_t roff = (uint32_t)(lane >> 3) * 4096u + (uint32_t)r * 128u + (uint32_t)(((lane & 7) ^ (r & 7)) << 4);
        float4 y = *reinterpret_cast<const float4 *>(raw + roff);
        float4 o = y;
        if (P.a_mode == CODA_A32_BN_BWD) {
          const float4 d = *reinterpret_cast<const float4 *>(raw + RAW_A + roff);
          o.x = (fmaf(y.x, sa.x, ta.x) > 0.f ? sa.x * d.x : 0.f) + fmaf(y.x, al.x, be.x);
          o.y = (fmaf(y.y, sa.y, ta.y) > 0.f ? sa.y * d.y : 0.f) + fmaf(y.y, al.y, be.y);
          o.z = (fmaf(y.z, sa.z, ta.z) > 0.f ? sa.z * d.z : 0.f) + fmaf(y.z, al.z, be.z);
          o.w = (fmaf(y.w, sa.w, ta.w) > 0.f ? sa.w * d.w : 0.f) + fmaf(y.w, al.w, be.w);
        } else if (P.a_mode == CODA_A32_BN_BWD_POOLED_PRE) {
          const int gi = rem0 + r;
          const float4 d = *reinterpret_cast<const float4 *>(raw + 2 * RAW_A + RAW_B + lane * 16);
          const uchar4 id = *reinterpret_cast<const uchar4 *>(raw + 2 * RAW_A + RAW_B + 512 + lane * 4);
          o.x = (id.x == gi ? d.x : 0.f) + fmaf(y.x, al.x, be.x);
          o.y = (id.y == gi ? d.y : 0.f) + fmaf(y.y, al.y, be.y);
          o.z = (id.z == gi ? d.z : 0.f) + fmaf(y.z, al.z, be.z);
          o.w = (id.w == gi ? d.w : 0.f) + fmaf(y.w, al.w, be.w);
        } else if (P.a_mode == CODA_A32_BN_BWD_POOLED) {
          const int gi = rem0 + r;
          const float4 d = *reinterpret_cast<const float4 *>(raw + 2 * RAW_A + RAW_B + lane * 16);
          const uchar4 id = *reinterpret_cast<const uchar4 *>(raw + 2 * RAW_A + RAW_B + 512 + lane * 4);
          o.x = ((id.x == gi && fmaf(y.x, sa.x, ta.x) > 0.f) ? sa.x * d.x : 0.f) + fmaf(y.x, al.x, be.x);
          o.y = ((id.y == gi && fmaf(y.y, sa.y, ta.y) > 0.f) ? sa.y * d.y : 0.f) + fmaf(y.y, al.y, be.y);
          o.z = ((id.z == gi && fmaf(y.z, sa.z, ta.z) > 0.f) ? sa.z * d.z : 0.f) + fmaf(y.z, al.z, be.z);
          o.w = ((id.w == gi && fmaf(y.w, sa.w, ta.w) > 0.f) ? sa.w * d.w : 0.f) + fmaf(y.w, al.w, be.w);
        }
        if (tail && grow >= P.rows) o = make_float4(0.f, 0.f, 0.f, 0.f);     // padding rows of the last slab
        if (want_colsum) { csum.x += o.x; csum.y += o.y; csum.z += o.z; csum.w += o.w; }
        // destination: box = column / 64, 16-byte chunk = (column % 64) / 8 swizzled by the row, half = (column % 8) / 4
        const int col = lane * 4;
        store_planes4(o, pl + (col >> 6) * (BKR * 128) + r * 128 + ((((col & 63) >> 3) ^ (r & 7)) << 4) + ((col & 7) >> 2) * 8,
                      PL_A);
      }
      // ---- B slab
#pragma unroll
      for (int j = 0; j < BKR / (TW * B_RPP); ++j) {
        const int r = (tw + j * TW) * B_RPP + brow_off;
        const long long grow = r0 + r;
        const uint32_t roff = (uint32_t)(bch >> 3) * 4096u + (uint32_t)r * 128u + (uint32_t)(((bch & 7) ^ (r & 7)) << 4);
        float4 v = *reinterpret_cast<const float4 *>(raw + 2 * RAW_A + roff);
        if (P.b_mode == CODA_A32_AFFINE_RELU) {
          v.x = fmaxf(fmaf(v.x, sb.x, tb.x), 0.f); v.y = fmaxf(fmaf(v.y, sb.y, tb.y), 0.f);
          v.z = fmaxf(fmaf(v.z, sb.z, tb.z), 0.f); v.w = fmaxf(fmaf(v.w, sb.w, tb.w), 0.f);
        }
        if (tail && grow >= P.rows) v = make_float4(0.f, 0.f, 0.f, 0.f);
        const int col = bch * 4;
        store_planes4(v, pl + NS * PL_A + (col >> 6) * (BKR * 128) + r * 128 + ((((col & 63) >> 3) ^ (r & 7)) << 4) +
                             ((col & 7) >> 2) * 8,
                      PL_B);
      }
      fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core's async-proxy reads
      __syncwarp();
      if (lane == 0) mbar_arrive(&raw_empty[rs]);
      bar_sync(1, 256);              // both operand slabs are complete in shared memory
      // plane products: lo*hi, hi*lo, hi*hi (small terms first); the warpgroup's 64 rows are the A slab's box wg
      acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        const int pa = p == 0 ? 1 : 0, pb = p == 1 ? 1 : 0;
        const uint64_t ad = gmma_desc_mn_sw128(pl + pa * PL_A + wg * (BKR * 128), BKR * 128);
        const uint64_t bd = gmma_desc_mn_sw128(pl + NS * PL_A + pb * PL_B, BKR * 128);
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
  // ===== epilogue: registers -> C, or (split-K) -> the split's scratch slot, added in split order by splitk_reduce_kernel
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

template <int BN>
int launch_tn32(const TN32Maps &maps, TN32Params P, float *c, long long ldc, cudaStream_t s) {
  constexpr size_t smem = (size_t)RAW_STAGES * (2 * BKR * BM * 4 + BKR * BN * 4 + 1024) +
                          (size_t)PL_STAGES * NS * (BKR * BM * 2 + BKR * BN * 2) + 1024;
  static_assert(smem <= 227 * 1024, "smem budget");
  auto kern = gemm_tn32_kernel<BN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  static int num_sms = 0;
  if (!num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (num_sms <= 0) num_sms = 132;
  }
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
    const long long total = (long long)P.m * P.n;
    const long long blocks = (total + 255) / 256;
    splitk_reduce_kernel<<<(unsigned)(blocks < 8 * num_sms ? blocks : 8 * num_sms), 256, 0, s>>>(
        P.partial, ksplit, P.m, P.n, 1, BM, BN, nullptr, c, ldc, 0);
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
