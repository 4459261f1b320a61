// Fused multi-head attention BACKWARD for H100 (sm_90a), head dim 64 (3DETR encoder, CLIP) and 128
// (3DETR decoder).  Two wgmma kernels; the (Lq x Lk) probability / score-gradient tiles never leave
// the SM: they are produced in registers from the score accumulators and handed back to the tensor core as
// register A operands.
//
//   attn_bwd_dq_kernel   CTA = (bh, 64 NWG queries); loop over 64-key tiles j
//        S_j  = Qs K_j^T              dP_j = dO V_j^T           (register accumulators, 64 x 64 per warpgroup)
//        dS_j = P_j o (m_j o dP_j - D)    with P_j = exp(S_j - LSE), m = dropout factor, D = rowsum(dO o O)
//        dQ  += dS_j K_j              (dS_j from registers; K_j as an MN-major B operand -- the same smem tile
//                                      that served S_j; accumulated over j, scaled at the end)
//   attn_bwd_dkv_kernel  CTA = (bh, 64 NWG keys); loop over 64-query tiles i
//        S_i^T  = K Qs_i^T            dP_i^T = V dO_i^T
//        P~_i^T = P_i^T o m           dS_i^T = P_i^T o (m o dP_i^T - D_i)
//        dV += P~_i^T dO_i            dK += dS_i^T Qs_i         (A from registers, dO_i / Qs_i MN-major from the
//                                      tiles that served the scores; accumulated over i)
//
// S is recomputed in both kernels so that every accumulation stays inside one CTA: no atomics, deterministic.
// Operands are split-bf16 planes like the forward; the backward uses 2 planes (3 cross products, ~16 mantissa
// bits), enough for the 2e-3 gradient parity bar.  Only row-major packs of q, k, v, dO are needed (no transposed
// copies).  Head dim 128 runs one warpgroup per CTA: its accumulators (dK and dV, or dQ, plus S and dP) need the
// register file of a one-warpgroup CTA.
// Optional attention mask (bit-packed, 1 = key not visible to query; MaskedTransformerEncoder of the reference,
// models/transformer.py:146-211): one 64-bit word per (row, 64-column tile).
#include "../../include/coda_attention.h"
#include "attention_common.cuh"

using namespace coda;
using namespace coda::attn;

namespace {

constexpr int NS = 2;           // planes per operand in the backward
constexpr int NPROD = 3;

// D[bh][q] = sum_d dO * O   (both (Lq, B, H*hd)); one warp per (q, b, h)
__global__ void __launch_bounds__(256)
bwd_delta_kernel(int Lq, int B, int H, int hd, const float *__restrict__ dout, const float *__restrict__ out,
                 float *__restrict__ delta) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= Lq * B * H) return;
  const int h = warp % H, b = (warp / H) % B, q = warp / (H * B);
  const size_t off = ((size_t)q * B + b) * H * hd + (size_t)h * hd;
  float s = 0.f;
  for (int d = lane; d < hd; d += 32) s += __ldg(dout + off + d) * __ldg(out + off + d);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) delta[(size_t)(b * H + h) * Lq + q] = s;
}

struct BwdMaps {
  CUtensorMap q[NS], k[NS], v[NS], dO[NS];
};

__device__ __forceinline__ float ex2_approx_b(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Shared-memory plan of both kernels: RES = the CTA's resident rows (two operands x NS planes x NWG 64-row boxes per
// 64 head-dim columns), then NST stages of the streamed 64-row tiles (two operands x NS planes).
template <int HD, int NWG>
struct BwdCfg {
  static constexpr int KB = HD / 64;
  static constexpr int BOX = 64 * 128;                // [64 x 64] bf16 box
  static constexpr int RES_PLANE = NWG * KB * BOX;    // one plane of one resident operand
  static constexpr int RES = 2 * NS * RES_PLANE;
  static constexpr int TILE_PLANE = KB * BOX;         // one plane of one streamed 64-row tile
  static constexpr int STAGE = 2 * NS * TILE_PLANE;
  static constexpr int NST_FIT = (220 * 1024 - RES) / STAGE;
  static constexpr int NST = NST_FIT > 4 ? 4 : NST_FIT;
  static constexpr int TOTAL = RES + NST * STAGE;
  static constexpr int THREADS = NWG * 128 + 32;
  static_assert(NST >= 1 && TOTAL + 1024 <= 227 * 1024, "smem budget");
};

// the two 64 x 64 score-side products X Y^T of one tile (X resident rows of the warpgroup, Y a streamed tile):
// s = X0 Y0^T, t = X1 Y1^T over NS planes x KB head-dim blocks
template <int KB>
__device__ __forceinline__ void scores2(float (&s)[32], float (&t)[32], const unsigned char *x0, const unsigned char *y0,
                                        const unsigned char *x1, const unsigned char *y1, int res_plane, int tile_plane) {
  acc_fence(s);
  acc_fence(t);
  wgmma_fence();
#pragma unroll
  for (int p = 0; p < NPROD; ++p)
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const int xo = a_pa(NS, p) * res_plane + kb * 8192, yo = a_pb(NS, p) * tile_plane + kb * 8192;
      const uint64_t ax = gmma_desc_k_sw128(x0 + xo), by = gmma_desc_k_sw128(y0 + yo);
      const uint64_t ax1 = gmma_desc_k_sw128(x1 + xo), by1 = gmma_desc_k_sw128(y1 + yo);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        Wgmma<64, false>::template ss<0, 0>(s, gmma_desc_advance(ax, kk * 32), gmma_desc_advance(by, kk * 32),
                                            (p | kb | kk) != 0);
        Wgmma<64, false>::template ss<0, 0>(t, gmma_desc_advance(ax1, kk * 32), gmma_desc_advance(by1, kk * 32),
                                            (p | kb | kk) != 0);
      }
    }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(s);
  acc_fence(t);
}

// ====================================================================== dQ
template <int HD, int NWG>
__global__ void __launch_bounds__(BwdCfg<HD, NWG>::THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ BwdMaps maps, int Lq, int Lk, int B, int H, float scale,
                   const float *__restrict__ lse, const float *__restrict__ delta, float *__restrict__ dq,
                   long long ld_dq, const unsigned long long *__restrict__ mask_q, float drop_p, uint32_t seed,
                   const uint32_t *__restrict__ seed_dev) {
  using C = BwdCfg<HD, NWG>;
  constexpr int KB = C::KB, NST = C::NST;
  if (seed_dev) seed += __ldg(seed_dev);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t q_full, kv_full[NST], kv_empty[NST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 64 * NWG, bh = blockIdx.y;
  const int ntiles = (Lk + 63) / 64;
  // resident: Qs planes at 0, dO planes at NS * RES_PLANE;  stage: K planes, then V planes
  if (threadIdx.x == 0) {
    mbar_init(&q_full, 1);
    for (int i = 0; i < NST; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], NWG); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp == NWG * 4) {
    // ===== TMA producer (warp-uniform control flow, one elected lane issues) =====
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(&q_full, (uint32_t)C::RES);
#pragma unroll
      for (int p = 0; p < NS; ++p)
#pragma unroll
        for (int w = 0; w < NWG; ++w)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            const int off = p * C::RES_PLANE + (w * KB + kb) * C::BOX;
            tma_load_3d(smem + off, &maps.q[p], &q_full, kb * 64, q0 + 64 * w, bh);
            tma_load_3d(smem + NS * C::RES_PLANE + off, &maps.dO[p], &q_full, kb * 64, q0 + 64 * w, bh);
          }
    }
    __syncwarp();
    for (int j = 0; j < ntiles; ++j) {
      const int st = j % NST;
      mbar_wait(&kv_empty[st], ((uint32_t)(j / NST) & 1u) ^ 1u);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&kv_full[st], (uint32_t)C::STAGE);
        unsigned char *sb = smem + C::RES + st * C::STAGE;
#pragma unroll
        for (int p = 0; p < NS; ++p)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            tma_load_3d(sb + (p * KB + kb) * C::BOX, &maps.k[p], &kv_full[st], kb * 64, j * 64, bh);
            tma_load_3d(sb + NS * C::TILE_PLANE + (p * KB + kb) * C::BOX, &maps.v[p], &kv_full[st], kb * 64, j * 64, bh);
          }
      }
      __syncwarp();
    }
    return;
  }

  const int w = warp >> 2, wl = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int qrow[2] = {q0 + 64 * w + wl * 16 + g, q0 + 64 * w + wl * 16 + g + 8};
  float lse2[2], d_r[2];
  const unsigned long long *mrow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const bool valid = qrow[i] < Lq;
    lse2[i] = (valid ? __ldg(lse + (size_t)bh * Lq + qrow[i]) : 0.f) * LOG2E;
    d_r[i] = valid ? __ldg(delta + (size_t)bh * Lq + qrow[i]) : 0.f;
    mrow[i] = mask_q ? mask_q + ((size_t)(bh / H) * Lq + (valid ? qrow[i] : 0)) * (size_t)ntiles : nullptr;
  }
  const bool dropout = drop_p > 0.f;
  const uint32_t thresh32 = drop_thresh32(drop_p);
  const float keep_scale = dropout ? 1.0f / (1.0f - drop_p) : 1.0f;
  const unsigned char *qs = smem + w * KB * C::BOX, *dos = qs + NS * C::RES_PLANE;
  float dq_acc[HD / 2];
  acc_zero(dq_acc);
  mbar_wait(&q_full, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int st = j % NST;
    const unsigned char *ks = smem + C::RES + st * C::STAGE, *vs = ks + NS * C::TILE_PLANE;
    mbar_wait(&kv_full[st], (uint32_t)(j / NST) & 1u);
    float sacc[32], pacc[32];
    scores2<KB>(sacc, pacc, qs, ks, dos, vs, C::RES_PLANE, C::TILE_PLANE);
    const int kvalid = Lk - j * 64;
    uint32_t af[4][NS][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t ts = dropout ? drop_tile_seed(seed, (uint32_t)bh, (uint32_t)qrow[i], (uint32_t)j) : 0u;
      const unsigned long long mb = mrow[i] ? __ldg(mrow[i] + j) : 0ull;
      const bool valid_row = qrow[i] < Lq;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        float ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = c * 8 + 2 * t4 + e;
          const bool vis = col < kvalid && valid_row && !((mb >> col) & 1ull);
          const float p = vis ? ex2_approx_b(fmaf(sacc[c * 4 + i * 2 + e], LOG2E, -lse2[i])) : 0.f;
          float dp = pacc[c * 4 + i * 2 + e];
          if (dropout) dp = (ts * kLcgJump.a[col] + kLcgJump.c[col] >= thresh32) ? dp * keep_scale : 0.f;
          ds[e] = p * (dp - d_r[i]);
        }
        uint32_t wv[NS];
        split_pair<NS>(ds[0], ds[1], wv);
#pragma unroll
        for (int pl = 0; pl < NS; ++pl) af[c >> 1][pl][(c & 1) * 2 + i] = wv[pl];
      }
    }
    acc_fence(dq_acc);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < NPROD; ++p) {
      const uint64_t bk = gmma_desc_mn_sw128(ks + a_pb(NS, p) * C::TILE_PLANE);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)   // 16 keys: 16 rows x 128 B of K_j
        Wgmma<HD, false>::template rs<1>(dq_acc, af[kk][a_pa(NS, p)], gmma_desc_advance(bk, kk * 16 * 128), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(dq_acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
  }
  const int b = bh / H, h = bh - b * H;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (qrow[i] >= Lq) continue;
    float *orow = dq + ((size_t)qrow[i] * B + b) * (size_t)ld_dq + (size_t)h * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c)
      *reinterpret_cast<float2 *>(orow + c * 8 + 2 * t4) =
          make_float2(dq_acc[c * 4 + i * 2] * scale, dq_acc[c * 4 + i * 2 + 1] * scale);
  }
}

// ====================================================================== dK, dV
template <int HD, int NWG>
__global__ void __launch_bounds__(BwdCfg<HD, NWG>::THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ BwdMaps maps, int Lq, int Lk, int B, int H,
                    const float *__restrict__ lse, const float *__restrict__ delta, float *__restrict__ dk,
                    float *__restrict__ dv, long long ld_dk, long long ld_dv,
                    const unsigned long long *__restrict__ mask_k, float drop_p, uint32_t seed,
                    const uint32_t *__restrict__ seed_dev) {
  using C = BwdCfg<HD, NWG>;
  constexpr int KB = C::KB, NST = C::NST;
  if (seed_dev) seed += __ldg(seed_dev);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t kv_full, q_full[NST], q_empty[NST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * 64 * NWG, bh = blockIdx.y;
  const int ntiles = (Lq + 63) / 64;
  // resident: K planes at 0, V planes at NS * RES_PLANE;  stage: Qs planes, then dO planes
  if (threadIdx.x == 0) {
    mbar_init(&kv_full, 1);
    for (int i = 0; i < NST; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], NWG); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp == NWG * 4) {
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(&kv_full, (uint32_t)C::RES);
#pragma unroll
      for (int p = 0; p < NS; ++p)
#pragma unroll
        for (int w = 0; w < NWG; ++w)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            const int off = p * C::RES_PLANE + (w * KB + kb) * C::BOX;
            tma_load_3d(smem + off, &maps.k[p], &kv_full, kb * 64, k0 + 64 * w, bh);
            tma_load_3d(smem + NS * C::RES_PLANE + off, &maps.v[p], &kv_full, kb * 64, k0 + 64 * w, bh);
          }
    }
    __syncwarp();
    for (int i = 0; i < ntiles; ++i) {
      const int st = i % NST;
      mbar_wait(&q_empty[st], ((uint32_t)(i / NST) & 1u) ^ 1u);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&q_full[st], (uint32_t)C::STAGE);
        unsigned char *sb = smem + C::RES + st * C::STAGE;
#pragma unroll
        for (int p = 0; p < NS; ++p)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            tma_load_3d(sb + (p * KB + kb) * C::BOX, &maps.q[p], &q_full[st], kb * 64, i * 64, bh);
            tma_load_3d(sb + NS * C::TILE_PLANE + (p * KB + kb) * C::BOX, &maps.dO[p], &q_full[st], kb * 64, i * 64, bh);
          }
      }
      __syncwarp();
    }
    return;
  }

  const int w = warp >> 2, wl = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int krow[2] = {k0 + 64 * w + wl * 16 + g, k0 + 64 * w + wl * 16 + g + 8};
  const unsigned long long *mrow[2];
  uint32_t ja[2], jc[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mrow[i] = mask_k ? mask_k + ((size_t)(bh / H) * Lk + (krow[i] < Lk ? krow[i] : 0)) * (size_t)ntiles : nullptr;
    ja[i] = kLcgJump.a[krow[i] & 63];   // this key's position in its 64-key tile
    jc[i] = kLcgJump.c[krow[i] & 63];
  }
  const uint32_t ktile = (uint32_t)((k0 >> 6) + w);   // both rows of a thread lie in the warpgroup's key tile
  const bool dropout = drop_p > 0.f;
  const uint32_t thresh32 = drop_thresh32(drop_p);
  const float keep_scale = dropout ? 1.0f / (1.0f - drop_p) : 1.0f;
  const unsigned char *kres = smem + w * KB * C::BOX, *vres = kres + NS * C::RES_PLANE;
  float dk_acc[HD / 2], dv_acc[HD / 2];
  acc_zero(dk_acc);
  acc_zero(dv_acc);
  mbar_wait(&kv_full, 0);
  for (int it = 0; it < ntiles; ++it) {
    const int st = it % NST;
    const unsigned char *qs = smem + C::RES + st * C::STAGE, *dos = qs + NS * C::TILE_PLANE;
    // the per-query values of this thread's 16 columns: log-sum-exp (log2 units), D, dropout stream seeds
    float lse16[16], dl16[16];
    uint32_t sd16[16];
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int qi = it * 64 + c * 8 + 2 * t4 + e;
        const bool ok = qi < Lq;
        lse16[c * 2 + e] = ok ? __ldg(lse + (size_t)bh * Lq + qi) * LOG2E : 0.f;
        dl16[c * 2 + e] = ok ? __ldg(delta + (size_t)bh * Lq + qi) : 0.f;
        sd16[c * 2 + e] = dropout ? drop_tile_seed(seed, (uint32_t)bh, (uint32_t)qi, ktile) : 0u;
      }
    mbar_wait(&q_full[st], (uint32_t)(it / NST) & 1u);
    float sacc[32], pacc[32];
    scores2<KB>(sacc, pacc, kres, qs, vres, dos, C::RES_PLANE, C::TILE_PLANE);
    const int qvalid = Lq - it * 64;
    uint32_t pf[4][NS][4], sf[4][NS][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const unsigned long long mb = mrow[i] ? __ldg(mrow[i] + it) : 0ull;
      const bool valid_row = krow[i] < Lk;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        float pt[2], ds[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = c * 8 + 2 * t4 + e;
          const bool vis = col < qvalid && valid_row && !((mb >> col) & 1ull);
          const float p = vis ? ex2_approx_b(fmaf(sacc[c * 4 + i * 2 + e], LOG2E, -lse16[c * 2 + e])) : 0.f;
          const float dp = pacc[c * 4 + i * 2 + e];
          float m = 1.0f;
          if (dropout) m = (sd16[c * 2 + e] * ja[i] + jc[i] >= thresh32) ? keep_scale : 0.f;
          pt[e] = p * m;
          ds[e] = p * (dp * m - dl16[c * 2 + e]);
        }
        uint32_t wp[NS], ws[NS];
        split_pair<NS>(pt[0], pt[1], wp);
        split_pair<NS>(ds[0], ds[1], ws);
#pragma unroll
        for (int pl = 0; pl < NS; ++pl) {
          pf[c >> 1][pl][(c & 1) * 2 + i] = wp[pl];
          sf[c >> 1][pl][(c & 1) * 2 + i] = ws[pl];
        }
      }
    }
    acc_fence(dv_acc);
    acc_fence(dk_acc);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < NPROD; ++p) {
      const uint64_t bo = gmma_desc_mn_sw128(dos + a_pb(NS, p) * C::TILE_PLANE);
      const uint64_t bq = gmma_desc_mn_sw128(qs + a_pb(NS, p) * C::TILE_PLANE);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // 16 queries: 16 rows x 128 B of dO_i / Qs_i
        Wgmma<HD, false>::template rs<1>(dv_acc, pf[kk][a_pa(NS, p)], gmma_desc_advance(bo, kk * 16 * 128), 1);
        Wgmma<HD, false>::template rs<1>(dk_acc, sf[kk][a_pa(NS, p)], gmma_desc_advance(bq, kk * 16 * 128), 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(dv_acc);
    acc_fence(dk_acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&q_empty[st]);
  }
  const int b = bh / H, h = bh - b * H;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (krow[i] >= Lk) continue;
    float *vrow = dv + ((size_t)krow[i] * B + b) * (size_t)ld_dv + (size_t)h * HD;
    float *krw = dk + ((size_t)krow[i] * B + b) * (size_t)ld_dk + (size_t)h * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      *reinterpret_cast<float2 *>(vrow + c * 8 + 2 * t4) = make_float2(dv_acc[c * 4 + i * 2], dv_acc[c * 4 + i * 2 + 1]);
      *reinterpret_cast<float2 *>(krw + c * 8 + 2 * t4) = make_float2(dk_acc[c * 4 + i * 2], dk_acc[c * 4 + i * 2 + 1]);
    }
  }
}

template <int HD>
int launch_bwd(const BwdMaps &mq, const BwdMaps &mk, int b, int h, int lq, int lk, float scale, const float *lse,
               const float *delta, float *dq, float *dk, float *dv, long long ld_dq, long long ld_dk, long long ld_dv,
               const unsigned long long *mask_q, const unsigned long long *mask_k, float dropout_p, unsigned int seed,
               const unsigned int *seed_dev, cudaStream_t s) {
  constexpr int NWG = HD == 64 ? 2 : 1;
  using C = BwdCfg<HD, NWG>;
  static bool configured = false;  // once per template instance
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_dq_kernel<HD, NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         C::TOTAL + 1024);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(attn_bwd_dkv_kernel<HD, NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::TOTAL + 1024);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int bh = b * h, rows = 64 * NWG;
  attn_bwd_dq_kernel<HD, NWG><<<dim3((lq + rows - 1) / rows, bh), C::THREADS, C::TOTAL + 1024, s>>>(
      mq, lq, lk, b, h, scale, lse, delta, dq, ld_dq, mask_q, dropout_p, seed, seed_dev);
  attn_bwd_dkv_kernel<HD, NWG><<<dim3((lk + rows - 1) / rows, bh), C::THREADS, C::TOTAL + 1024, s>>>(
      mk, lq, lk, b, h, lse, delta, dk, dv, ld_dk, ld_dv, mask_k, dropout_p, seed, seed_dev);
  return launch_status();
}

}  // namespace

extern "C" {

long long coda_attention_bwd_workspace_bytes(int b, int h, int lq, int lk, int hd) {
  const long long bh = (long long)b * h;
  // q, dO rows; k, v rows (NS bf16 planes each) + delta
  return 2LL * NS * bh * hd * (2LL * lq + 2LL * lk) + 4LL * bh * lq + 4096;
}

int coda_attention_bwd(int b, int h, int lq, int lk, int hd, float scale, const float *q, const float *k,
                       const float *v, const float *out, const float *dout, const float *lse, float *dq,
                       float *dk, float *dv, float dropout_p, unsigned int seed, const unsigned int *seed_dev,
                       void *workspace, void *stream) {
  const long long e = (long long)h * hd;
  return coda_attention_bwd_ex(b, h, lq, lk, hd, scale, q, k, v, e, e, e, out, dout, lse, dq, dk, dv, e, e, e, nullptr,
                               nullptr, dropout_p, seed, seed_dev, workspace, stream);
}

int coda_attention_bwd_ex(int b, int h, int lq, int lk, int hd, float scale, const float *q, const float *k,
                          const float *v, long long ld_q, long long ld_k, long long ld_v, const float *out,
                          const float *dout, const float *lse, float *dq, float *dk, float *dv, long long ld_dq,
                          long long ld_dk, long long ld_dv, const unsigned long long *mask_q,
                          const unsigned long long *mask_k, float dropout_p, unsigned int seed,
                          const unsigned int *seed_dev, void *workspace, void *stream) {
  if ((hd != 64 && hd != 128) || b < 0 || h <= 0 || lq <= 0 || lk <= 0 || (long long)b * h > 65535) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!q || !k || !v || !out || !dout || !lse || !dq || !dk || !dv || !workspace) return CODA_EINVAL;
  if (dropout_p < 0.f || dropout_p >= 1.f) return CODA_EINVAL;
  if ((mask_q == nullptr) != (mask_k == nullptr)) return CODA_EINVAL;
  {
    const long long e0 = (long long)h * hd;
    if (ld_q < e0 || ld_k < e0 || ld_v < e0 || ld_dq < e0 || ld_dk < e0 || ld_dv < e0) return CODA_EINVAL;
    if ((ld_q | ld_k | ld_v | ld_dq | ld_dk | ld_dv) & 3) return CODA_EINVAL;
    if ((((uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) & 15) != 0) return CODA_EINVAL;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int bh = b * h;
  __nv_bfloat16 *w = (__nv_bfloat16 *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  __nv_bfloat16 *qp = w;                                   w += (size_t)NS * bh * lq * hd;
  __nv_bfloat16 *dop = w;                                  w += (size_t)NS * bh * lq * hd;
  __nv_bfloat16 *kp = w;                                   w += (size_t)NS * bh * lk * hd;
  __nv_bfloat16 *vp = w;                                   w += (size_t)NS * bh * lk * hd;
  float *delta = (float *)(((uintptr_t)w + 255) & ~(uintptr_t)255);
  if ((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dout) & 15) != 0) return CODA_EINVAL;
  PackJobs jobs = {};
  const long long e = (long long)h * hd;
  jobs.job[0] = {q, qp, lq, scale, ld_q};
  jobs.job[1] = {dout, dop, lq, 1.0f, e};
  jobs.job[2] = {k, kp, lk, 1.0f, ld_k};
  jobs.job[3] = {v, vp, lk, 1.0f, ld_v};
  const long long t4 = (long long)(lq > lk ? lq : lk) * bh * hd / 4;
  pack_rows_multi_kernel<NS, false><<<dim3((unsigned)((t4 + 255) / 256), 4), 256, 0, s>>>(jobs, b, h, hd);
  bwd_delta_kernel<<<(unsigned)(((long long)lq * bh * 32 + 255) / 256), 256, 0, s>>>(lq, b, h, hd, dout, out, delta);
  int st = launch_status();
  if (st != CODA_OK) return st;

  BwdMaps mq, mk;  // every box is 64 rows: resident rows are loaded one warpgroup slice at a time
  for (int p = 0; p < NS; ++p) {
    const size_t oq = (size_t)p * bh * lq * hd, ok = (size_t)p * bh * lk * hd;
#define MAP(dst, base, rows, box) \
  if ((st = make_tmap_k_major_16b(&(dst), (base), 0, hd, (rows), bh, hd, (long long)(rows) * hd, (box))) != CODA_OK) return st
    MAP(mq.q[p], qp + oq, lq, 64);
    MAP(mq.dO[p], dop + oq, lq, 64);
    MAP(mq.k[p], kp + ok, lk, 64);
    MAP(mq.v[p], vp + ok, lk, 64);
    MAP(mk.k[p], kp + ok, lk, 64);
    MAP(mk.v[p], vp + ok, lk, 64);
    MAP(mk.q[p], qp + oq, lq, 64);
    MAP(mk.dO[p], dop + oq, lq, 64);
#undef MAP
  }
  if (hd == 64)
    return launch_bwd<64>(mq, mk, b, h, lq, lk, scale, lse, delta, dq, dk, dv, ld_dq, ld_dk, ld_dv, mask_q, mask_k,
                          dropout_p, seed, seed_dev, s);
  return launch_bwd<128>(mq, mk, b, h, lq, lk, scale, lse, delta, dq, dk, dv, ld_dq, ld_dk, ld_dv, mask_q, mask_k,
                         dropout_p, seed, seed_dev, s);
}

}  // extern "C"
