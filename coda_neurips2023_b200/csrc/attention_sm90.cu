// Fused multi-head attention forward for H100 (sm_90a): S = Q K^T and O = P V on wgmma tensor cores with
// register accumulators, operands staged by TMA into 128B-swizzled shared memory, online softmax in registers.
// The (Lq x Lk) probability matrix never leaves the SM.  C-ABI in include/coda_attention.h.
//
// Numerics: q (pre-scaled), k, v are fp32; each is split into NSPLIT bf16 planes
// (x = p0 + p1 (+ p2)) by pack_rows_multi_kernel and the 1 / 3 / 6 significant cross
// products are accumulated in fp32 -- fp32-class results at bf16 tensor-core rate
// (same scheme as gemm_sm90.cu).  P (in [0, 1]) carries at most two planes.  q is
// packed with scale * log2(e), so the scores are in log2 units and the softmax is one
// ex2 per element; the log-sum-exp is returned in natural-log units.
//
// One CTA = one (batch*head, 64 * NWG query tile); loop over 64-key tiles:
//   last warp          : TMA producer of Q (once) and of K_j / V_j (row-major tiles; V_j is consumed as an
//                        MN-major B operand: no transposed copy of V exists)
//   warpgroup w < NWG  : query rows [64 w, +64): S_j = Q K_j^T (wgmma, both operands from shared memory), online
//                        softmax on the accumulator registers, P_j planes re-used in registers as the A operand of
//                        O_j = P_j V_j (wgmma with register A), o = o * alpha + O_j kept in registers.
#include <math.h>

#include "../../include/coda_attention.h"
#include "attention_common.cuh"

using namespace coda;
using namespace coda::attn;

namespace {

// materialised keep-mask * 1/(1-p) for the interim (cuBLAS) backward: mult[bh][q][k] in {0, 1/(1-p)}
__global__ void __launch_bounds__(256)
dropout_mult_kernel(long long total, int lq, int lk, uint32_t seed, const uint32_t *__restrict__ seed_dev,
                    uint32_t thresh32, float keep_scale, float *__restrict__ mult) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  if (seed_dev) seed += __ldg(seed_dev);
  const uint32_t k = (uint32_t)(i % lk);
  const long long t = i / lk;
  const uint32_t q = (uint32_t)(t % lq), bh = (uint32_t)(t / lq);
  mult[i] = drop_keep(seed, bh, q, k, thresh32) ? keep_scale : 0.f;
}

// Attention masks travel bit-packed: bits[b][row][tile] (one 64-bit word per 64 columns), bit c set = column
// 64 * tile + c is NOT visible from that row (torch's boolean attn_mask convention).  The forward and the dQ kernel
// index rows by query, the dK/dV kernel by key (the transposed packing), so every softmax thread reads one word
// per tile.  rows / cols and the strides are in the orientation being packed.
__global__ void __launch_bounds__(128)
mask_pack_kernel(int B, int rows, int cols, const unsigned char *__restrict__ mask, long long stride_b,
                 long long stride_r, long long stride_c, unsigned long long *__restrict__ bits) {
  const int nt = (cols + 63) / 64;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * rows * nt) return;
  const int t = (int)(i % nt);
  const long long br = i / nt;
  const int r = (int)(br % rows), b = (int)(br / rows);
  const unsigned char *src = mask + (size_t)b * stride_b + (size_t)r * stride_r;
  unsigned long long w = 0;
  for (int c = 0; c < 64; ++c) {
    const int col = t * 64 + c;
    if (col < cols && __ldg(src + (size_t)col * stride_c)) w |= 1ull << c;
  }
  bits[i] = w;
}

// Radius mask of the reference's MaskedTransformerEncoder (models/transformer.py:155-162): point j is masked for
// point i when |x_i - x_j| >= radius (Euclidean, as torch.cdist).  Symmetric: one packing serves both orientations.
__global__ void __launch_bounds__(128)
mask_radius_kernel(int B, int L, const float *__restrict__ xyz, float radius, unsigned long long *__restrict__ bits) {
  const int nt = (L + 63) / 64;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * L * nt) return;
  const int t = (int)(i % nt);
  const long long br = i / nt;
  const int r = (int)(br % L), b = (int)(br / L);
  const float *base = xyz + (size_t)b * L * 3;
  const float x = __ldg(base + 3 * r), y = __ldg(base + 3 * r + 1), z = __ldg(base + 3 * r + 2);
  unsigned long long w = 0;
  for (int c = 0; c < 64; ++c) {
    const int col = t * 64 + c;
    if (col >= L) break;
    const float dx = x - __ldg(base + 3 * col), dy = y - __ldg(base + 3 * col + 1), dz = z - __ldg(base + 3 * col + 2);
    if (sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx))) >= radius) w |= 1ull << c;
  }
  bits[i] = w;
}

// half in -> ONE plane of half operands [b*h][L][hd] (scaled): the fp16 tower's q / k / v need a re-layout, not a split
__global__ void __launch_bounds__(256)
pack_rows_half_kernel(const __grid_constant__ PackJobs jobs, int B, int H, int hd) {
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
  uint2 raw = __ldg(reinterpret_cast<const uint2 *>(static_cast<const __half *>(jb.src) + off));
  if (jb.scale != 1.0f) {
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&raw.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&raw.y));
    const __half2 a = __floats2half2_rn(lo.x * jb.scale, lo.y * jb.scale), c = __floats2half2_rn(hi.x * jb.scale, hi.y * jb.scale);
    raw.x = *reinterpret_cast<const uint32_t *>(&a);
    raw.y = *reinterpret_cast<const uint32_t *>(&c);
  }
  __half *dst = reinterpret_cast<__half *>(jb.planes) + (((size_t)(b * H + h)) * jb.L + l) * hd + d;
  *reinterpret_cast<uint2 *>(dst) = raw;
}

// ------------------------------------------------------------------ the kernel
struct AttnMaps {
  CUtensorMap q[3], k[3], v[3];
};

// P lies in [0, 1] and is consumed once: two bf16 planes (relative error 2^-18) are enough even when
// q, k, v carry three, which drops one of the six cross products of O = P V.
__host__ __device__ constexpr int p_planes(int ns) { return ns == 3 ? 2 : ns; }
__host__ __device__ constexpr int pv_nprod(int ns) { return ns == 1 ? 1 : (ns == 2 ? 3 : 5); }
__host__ __device__ constexpr int pv_pa(int ns, int p) {  // plane of P, smallest terms first
  return ns == 1 ? 0 : ns == 2 ? (p == 0 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 0 : p == 2 ? 1 : 0);
}
__host__ __device__ constexpr int pv_pb(int ns, int p) {  // plane of V
  return ns == 1 ? 0 : ns == 2 ? (p == 1 ? 1 : 0) : (p == 0 ? 1 : p == 1 ? 2 : p == 2 ? 0 : p == 3 ? 1 : 0);
}

template <int HD, int NSPLIT, int NWG>
struct AttnCfg {
  static constexpr int KB = HD / 64;                       // 64-wide k-blocks of the head dim
  static constexpr int BOX = 64 * 128;                     // one [64 rows x 64] 16-bit box
  static constexpr int Q_BYTES = NSPLIT * NWG * KB * BOX;  // Q planes of the CTA's query rows
  static constexpr int KV_PLANE = KB * BOX;                // [64 keys x HD] per plane
  static constexpr int STAGE = 2 * NSPLIT * KV_PLANE;      // K_j and V_j
  static constexpr int NST_FIT = (220 * 1024 - Q_BYTES) / STAGE;
  static constexpr int NST = NST_FIT > 4 ? 4 : (NST_FIT < 1 ? 1 : NST_FIT);
  static constexpr int K_OFF = Q_BYTES;
  static constexpr int TOTAL = Q_BYTES + NST * STAGE;
  static constexpr int THREADS = NWG * 128 + 32;
  static_assert(TOTAL + 1024 <= 227 * 1024, "smem budget");
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// F16: the operand planes (and P) are IEEE half instead of bf16 -- the fp16 CLIP tower needs no split at all: one
// plane, one MMA per product, where two bf16 planes took three.
template <int HD, int NSPLIT, int NWG, bool F16 = false>
__global__ void __launch_bounds__(AttnCfg<HD, NSPLIT, NWG>::THREADS, 1)
attn_fwd_kernel(const __grid_constant__ AttnMaps maps, int Lq, int Lk, int B, int H, float *__restrict__ out,
                float *__restrict__ lse, float drop_p, uint32_t seed, const uint32_t *__restrict__ seed_dev,
                int out_half, const unsigned long long *__restrict__ mask_q) {
  using C = AttnCfg<HD, NSPLIT, NWG>;
  if (seed_dev) seed += __ldg(seed_dev);  // per-step counter kept on the device (CUDA-graph friendly)
  constexpr int KB = C::KB, NP = p_planes(NSPLIT), NST = C::NST;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = smem_align1024(smem_raw);
  __shared__ __align__(8) uint64_t q_full, kv_full[NST], kv_empty[NST];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 64 * NWG, bh = blockIdx.y;
  const int ntiles = (Lk + KT - 1) / KT;

  if (threadIdx.x == 0) {
    mbar_init(&q_full, 1);
    for (int i = 0; i < NST; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], NWG); }
    mbar_fence_init_cluster();
  }
  __syncthreads();

  if (warp == NWG * 4) {
    // ===== TMA producer =====
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(&q_full, (uint32_t)C::Q_BYTES);
#pragma unroll
      for (int p = 0; p < NSPLIT; ++p)
#pragma unroll
        for (int w = 0; w < NWG; ++w)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb)
            tma_load_3d(smem + ((p * NWG + w) * KB + kb) * C::BOX, &maps.q[p], &q_full, kb * 64, q0 + 64 * w, bh);
    }
    __syncwarp();
    for (int j = 0; j < ntiles; ++j) {
      const int st = j % NST;
      mbar_wait(&kv_empty[st], ((uint32_t)(j / NST) & 1u) ^ 1u);
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(&kv_full[st], (uint32_t)C::STAGE);
        unsigned char *sb = smem + C::K_OFF + st * C::STAGE;
#pragma unroll
        for (int p = 0; p < NSPLIT; ++p)
#pragma unroll
          for (int kb = 0; kb < KB; ++kb) {
            tma_load_3d(sb + (p * KB + kb) * C::BOX, &maps.k[p], &kv_full[st], kb * 64, j * KT, bh);
            tma_load_3d(sb + NSPLIT * C::KV_PLANE + (p * KB + kb) * C::BOX, &maps.v[p], &kv_full[st], kb * 64, j * KT, bh);
          }
      }
      __syncwarp();
    }
    return;
  }

  // ===== warpgroup w: query rows [64 w, +64); thread rows r0 = 16 wl + g and r0 + 8, columns 8 c + 2 t4 + {0, 1} =====
  const int w = warp >> 2, wl = warp & 3, g = lane >> 2, t4 = lane & 3;
  const int qrow[2] = {q0 + 64 * w + wl * 16 + g, q0 + 64 * w + wl * 16 + g + 8};
  float o_acc[HD / 2];
  acc_zero(o_acc);
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this thread's partial row sums
  const bool dropout = drop_p > 0.f;
  const uint32_t thresh32 = drop_thresh32(drop_p);
  const float keep_scale = dropout ? 1.0f / (1.0f - drop_p) : 1.0f;
  // attention mask: one 64-bit word per (batch, query row, key tile), bit c set = key c of the tile is not visible
  const unsigned long long *mrow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
    mrow[i] = mask_q ? mask_q + ((size_t)(bh / H) * Lq + (qrow[i] < Lq ? qrow[i] : 0)) * (size_t)ntiles : nullptr;
  const unsigned char *qs = smem + (size_t)w * KB * C::BOX;
  mbar_wait(&q_full, 0);

  for (int j = 0; j < ntiles; ++j) {
    const int st = j % NST;
    const unsigned char *ks = smem + C::K_OFF + st * C::STAGE;
    const unsigned char *vs = ks + NSPLIT * C::KV_PLANE;
    mbar_wait(&kv_full[st], (uint32_t)(j / NST) & 1u);
    float sacc[KT / 2];
    acc_fence(sacc);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < n_products(NSPLIT); ++p)
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const uint64_t ad = gmma_desc_k_sw128(qs + ((prod_a(NSPLIT, p) * NWG) * KB + kb) * C::BOX);
        const uint64_t bd = gmma_desc_k_sw128(ks + (prod_b(NSPLIT, p) * KB + kb) * C::BOX);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          Wgmma<KT, F16>::template ss<0, 0>(sacc, gmma_desc_advance(ad, kk * 32), gmma_desc_advance(bd, kk * 32),
                                            (p | kb | kk) != 0);
      }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(sacc);

    const int kvalid = Lk - j * KT;  // keys >= kvalid are padding (last tile only)
    float alpha[2], m_use[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const unsigned long long mb = mrow[i] ? __ldg(mrow[i] + j) : 0ull;
      float mloc = -INFINITY;
#pragma unroll
      for (int c = 0; c < KT / 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = c * 8 + 2 * t4 + e;
          float &x = sacc[c * 4 + i * 2 + e];
          if (col >= kvalid || ((mb >> col) & 1ull)) x = -INFINITY;
          mloc = fmaxf(mloc, x);
        }
      mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 1));
      mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 2));
      const float m_new = fmaxf(m_run[i], mloc);
      // a row whose keys so far are all masked keeps m = -inf; exponentials are then taken against 0 (all zero)
      m_use[i] = m_new == -INFINITY ? 0.f : m_new;
      alpha[i] = ex2_approx(m_run[i] - m_use[i]);  // m_run = -inf on the first tile -> 0
      m_run[i] = m_new;
    }
    // P_j = 2^(s - m) (dropped elements zeroed; the 1/(1-p) factor is applied once, at the end) -> A fragments
    uint32_t pf[KT / 16][NP][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float lsum = 0.f;
      const uint32_t ts = dropout ? drop_tile_seed(seed, (uint32_t)bh, (uint32_t)qrow[i], (uint32_t)j) : 0u;
#pragma unroll
      for (int c = 0; c < KT / 8; ++c) {
        float r[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = c * 8 + 2 * t4 + e;
          r[e] = ex2_approx(sacc[c * 4 + i * 2 + e] - m_use[i]);
          lsum += r[e];
          if (dropout && ts * kLcgJump.a[col] + kLcgJump.c[col] < thresh32) r[e] = 0.f;
        }
        uint32_t wv[NP];
        if constexpr (F16) {
          wv[0] = pack2<true>(r[0], r[1]);
        } else {
          split_pair<NP>(r[0], r[1], wv);
        }
        // key chunk c of 8: k-step c / 2, register (c & 1) * 2 + i
#pragma unroll
        for (int pl = 0; pl < NP; ++pl) pf[c >> 1][pl][(c & 1) * 2 + i] = wv[pl];
      }
      l_run[i] = l_run[i] * alpha[i] + lsum;
    }
    // O_j = P_j V_j in a fresh accumulator (cross products smallest first), then o = o * alpha + O_j
    float ot[HD / 2];
    acc_fence(ot);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < pv_nprod(NSPLIT); ++p) {
      const uint64_t bd = gmma_desc_mn_sw128(vs + pv_pb(NSPLIT, p) * C::KV_PLANE);
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk)
        Wgmma<HD, F16>::template rs<1>(ot, pf[kk][pv_pa(NSPLIT, p)], gmma_desc_advance(bd, kk * 16 * 128), (p | kk) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(ot);
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      o_acc[c * 4] = fmaf(o_acc[c * 4], alpha[0], ot[c * 4]);
      o_acc[c * 4 + 1] = fmaf(o_acc[c * 4 + 1], alpha[0], ot[c * 4 + 1]);
      o_acc[c * 4 + 2] = fmaf(o_acc[c * 4 + 2], alpha[1], ot[c * 4 + 2]);
      o_acc[c * 4 + 3] = fmaf(o_acc[c * 4 + 3], alpha[1], ot[c * 4 + 3]);
    }
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
  }

  // ===== epilogue: normalise, store (Lq, B, H*HD) and the log-sum-exp (natural-log units) =====
  const int b = bh / H, h = bh - b * H;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    if (qrow[i] >= Lq) continue;
    const float inv = keep_scale / l;
    const size_t ooff = ((size_t)qrow[i] * B + b) * (size_t)(H * HD) + (size_t)h * HD;
#pragma unroll
    for (int c = 0; c < HD / 8; ++c) {
      const int d = c * 8 + 2 * t4;
      const float v0 = o_acc[c * 4 + i * 2] * inv, v1 = o_acc[c * 4 + i * 2 + 1] * inv;
      if (out_half) *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(out) + ooff + d) = __floats2half2_rn(v0, v1);
      else *reinterpret_cast<float2 *>(out + ooff + d) = make_float2(v0, v1);
    }
    if (lse && t4 == 0) lse[(size_t)bh * Lq + qrow[i]] = m_run[i] * LN2 + logf(l);
  }
}

template <int HD, int NSPLIT, bool F16 = false>
int launch_attn(const AttnMaps &maps, int Lq, int Lk, int B, int H, float *out, float *lse, float drop_p, uint32_t seed,
                const uint32_t *seed_dev, cudaStream_t s, int out_half = 0, const unsigned long long *mask_q = nullptr) {
  static_assert(!F16 || NSPLIT == 1, "half operands are a single plane");
  // one warpgroup per CTA for short query sequences (the CLIP tower: 50 tokens) and for head dim 128 (its running
  // and per-tile O accumulators take the register file of a one-warpgroup CTA), two otherwise
  const bool one = Lq <= 64 || HD == 128;
  constexpr auto kern1 = attn_fwd_kernel<HD, NSPLIT, 1, F16>, kern2 = attn_fwd_kernel<HD, NSPLIT, 2, F16>;
  const auto kern = one ? kern1 : kern2;
  const int smem = (one ? AttnCfg<HD, NSPLIT, 1>::TOTAL : AttnCfg<HD, NSPLIT, 2>::TOTAL) + 1024;
  const int threads = one ? AttnCfg<HD, NSPLIT, 1>::THREADS : AttnCfg<HD, NSPLIT, 2>::THREADS;
  if (const int st = one ? raise_smem_limit<kern1>(smem) : raise_smem_limit<kern2>(smem)) return st;
  const int rows = one ? 64 : 128;
  const dim3 grid((Lq + rows - 1) / rows, B * H);
  kern<<<grid, threads, smem, s>>>(maps, Lq, Lk, B, H, out, lse, drop_p, seed, seed_dev, out_half, mask_q);
  return launch_status();
}

// ------------------------------------------------------------------ fp16 self-attention, 64 < L <= 256, hd 64
// The CLIP ViT-B/16 image tower (197 tokens).  One CTA per (crop, head): every Q, K and V tile of the sequence is
// loaded ONCE by TMA straight out of the fused in-projection output (L, N, ld) -- no pack pass, no workspace -- and
// stays resident in shared memory; the query tiles are spread over the warpgroups, and each walks all key tiles with
// the online softmax of attn_fwd_kernel.  The maps are 3-D: the head and head-dim indices are contiguous, so
// (h * 64 + d, token, crop) addresses q / k / v with a token stride of N * ld; TMA zero-fills tokens >= L.
struct HalfMaps {
  CUtensorMap q, k, v;
};

struct ResCfg {
  static constexpr int NT = 4;                  // tiles of 64 tokens: L <= 256
  static constexpr int NWG = 2;                 // warpgroups; warpgroup w takes query tiles w and w + 2
  static constexpr int BOX = 64 * 128;          // one [64 tokens x 64] half box
  static constexpr int Q_OFF = 0, K_OFF = NT * BOX, V_OFF = 2 * NT * BOX;
  static constexpr int TOTAL = 3 * NT * BOX;    // 96 KB: two CTAs per SM
  static constexpr int THREADS = NWG * 128;
};

// qk_scale = log2(e) / sqrt(hd), applied to the fp32 scores: the softmax works in base 2 (one ex2 per element)
__global__ void __launch_bounds__(ResCfg::THREADS, 2)
attn_fwd_half_resident_kernel(const __grid_constant__ HalfMaps maps, int L, int B, int H, float qk_scale,
                              __half *__restrict__ out) {
  using C = ResCfg;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = smem_align1024(smem_raw);
  __shared__ __align__(8) uint64_t q_full[C::NT], kv_full[C::NT];   // each completes once: phase parity 0

  const int bh = blockIdx.x, b = bh / H, h = bh - b * H;
  const int nt = (L + 63) / 64;
  if (threadIdx.x == 0) {
    for (int i = 0; i < C::NT; ++i) { mbar_init(&q_full[i], 1); mbar_init(&kv_full[i], 1); }
    mbar_fence_init_cluster();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // the first query tile of each warpgroup, then K_j / V_j in the order they are walked, then the second round
    auto load_q = [&](int t) {
      mbar_arrive_expect_tx(&q_full[t], (uint32_t)C::BOX);
      tma_load_3d(smem + C::Q_OFF + t * C::BOX, &maps.q, &q_full[t], h * 64, t * 64, b);
    };
    for (int t = 0; t < C::NWG && t < nt; ++t) load_q(t);
    for (int j = 0; j < nt; ++j) {
      mbar_arrive_expect_tx(&kv_full[j], (uint32_t)(2 * C::BOX));
      tma_load_3d(smem + C::K_OFF + j * C::BOX, &maps.k, &kv_full[j], h * 64, j * 64, b);
      tma_load_3d(smem + C::V_OFF + j * C::BOX, &maps.v, &kv_full[j], h * 64, j * 64, b);
    }
    for (int t = C::NWG; t < nt; ++t) load_q(t);
  }

  // thread rows r0 = 16 wl + g and r0 + 8 of the warpgroup's 64, columns 8 c + 2 t4 + {0, 1}
  const int w = threadIdx.x >> 7, wl = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  for (int t = w; t < nt; t += C::NWG) {
    const int qrow[2] = {t * 64 + wl * 16 + g, t * 64 + wl * 16 + g + 8};
    float o_acc[32];
    acc_zero(o_acc);
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // m_run: raw score units
    const unsigned char *qs = smem + C::Q_OFF + t * C::BOX;
    mbar_wait(&q_full[t], 0);
    for (int j = 0; j < nt; ++j) {
      const unsigned char *ks = smem + C::K_OFF + j * C::BOX, *vs = smem + C::V_OFF + j * C::BOX;
      mbar_wait(&kv_full[j], 0);
      float sacc[32];
      acc_fence(sacc);
      wgmma_fence();
      const uint64_t ad = gmma_desc_k_sw128(qs), bd = gmma_desc_k_sw128(ks);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        Wgmma<KT, true>::ss<0, 0>(sacc, gmma_desc_advance(ad, kk * 32), gmma_desc_advance(bd, kk * 32), kk != 0);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(sacc);

      const int kvalid = L - j * KT;  // keys >= kvalid are TMA's zero fill (last tile only)
      float alpha[2], mc[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float mloc = -INFINITY;
#pragma unroll
        for (int c = 0; c < KT / 8; ++c)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float &x = sacc[c * 4 + i * 2 + e];
            if (c * 8 + 2 * t4 + e >= kvalid) x = -INFINITY;
            mloc = fmaxf(mloc, x);
          }
        mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 1));
        mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 2));
        // tile 0 always holds a valid key (L > 0), so the running max is finite from the first tile on
        const float m_new = fmaxf(m_run[i], mloc);
        alpha[i] = ex2_approx((m_run[i] - m_new) * qk_scale);   // -inf on the first tile -> 0
        mc[i] = m_new * qk_scale;
        m_run[i] = m_new;
      }
      // P_j = 2^(s * qk_scale - m * qk_scale) -> fp16 A fragments (key chunk c of 8: k-step c / 2, register
      // (c & 1) * 2 + i)
      uint32_t pf[KT / 16][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float lsum = 0.f;
#pragma unroll
        for (int c = 0; c < KT / 8; ++c) {
          const float r0 = ex2_approx(fmaf(sacc[c * 4 + i * 2], qk_scale, -mc[i]));
          const float r1 = ex2_approx(fmaf(sacc[c * 4 + i * 2 + 1], qk_scale, -mc[i]));
          lsum += r0 + r1;
          pf[c >> 1][(c & 1) * 2 + i] = pack2<true>(r0, r1);
        }
        l_run[i] = l_run[i] * alpha[i] + lsum;
      }
      // o = o * alpha + P_j V_j: rescale the running accumulator in place, then accumulate into it
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        o_acc[c * 4] *= alpha[0];
        o_acc[c * 4 + 1] *= alpha[0];
        o_acc[c * 4 + 2] *= alpha[1];
        o_acc[c * 4 + 3] *= alpha[1];
      }
      acc_fence(o_acc);
      wgmma_fence();
      const uint64_t vd = gmma_desc_mn_sw128(vs);
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) Wgmma<64, true>::rs<1>(o_acc, pf[kk], gmma_desc_advance(vd, kk * 16 * 128), 1);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(o_acc);
    }
    // normalise and store rows < L of (L, B, H * 64) as half
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float l = l_run[i];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      if (qrow[i] >= L) continue;
      const float inv = 1.0f / l;
      __half *orow = out + ((size_t)qrow[i] * B + b) * (size_t)(H * 64) + (size_t)h * 64;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        *reinterpret_cast<__half2 *>(orow + c * 8 + 2 * t4) =
            __floats2half2_rn(o_acc[c * 4 + i * 2] * inv, o_acc[c * 4 + i * 2 + 1] * inv);
    }
  }
}

// q / k / v: (l, b, ld) half with the h * 64 head columns at the front of each row
int launch_attn_half_resident(int b, int h, int l, const void *q, const void *k, const void *v, long long ld_q,
                              long long ld_k, long long ld_v, __half *out, cudaStream_t s) {
  HalfMaps maps;
  const long long e = (long long)h * 64;
  int st = make_tmap_k_major_16b(&maps.q, q, 1, e, l, b, (long long)b * ld_q, ld_q, 64);
  if (st == CODA_OK) st = make_tmap_k_major_16b(&maps.k, k, 1, e, l, b, (long long)b * ld_k, ld_k, 64);
  if (st == CODA_OK) st = make_tmap_k_major_16b(&maps.v, v, 1, e, l, b, (long long)b * ld_v, ld_v, 64);
  if (st != CODA_OK) return st;
  constexpr auto kern = attn_fwd_half_resident_kernel;
  const int smem = ResCfg::TOTAL + 1024;
  if (const int r = raise_smem_limit<kern>(smem)) return r;
  kern<<<b * h, ResCfg::THREADS, smem, s>>>(maps, l, b, h, LOG2E / sqrtf(64.f), out);
  return launch_status();
}

}  // namespace

extern "C" {

long long coda_attention_workspace_bytes(int b, int h, int lq, int lk, int hd, int nsplit) {
  return 2LL * nsplit * b * h * ((long long)lq * hd + 2LL * lk * hd) + 1024;
}

static int attn_check(int b, int h, int lq, int lk, int hd, int nsplit) {
  if (b < 0 || h <= 0 || lq < 0 || lk <= 0 || (hd != 64 && hd != 128) || nsplit < 1 || nsplit > 3) return CODA_EINVAL;
  if ((long long)b * h > 65535) return CODA_EINVAL;
  return CODA_OK;
}

int coda_attention_pack_strided(int b, int h, int lq, int lk, int hd, int nsplit, float scale, const void *q,
                                const void *k, const void *v, long long ld_q, long long ld_k, long long ld_v,
                                int is_half, void *workspace, void *stream) {
  int st = attn_check(b, h, lq, lk, hd, nsplit);
  if (st != CODA_OK) return st;
  if (b == 0 || lq == 0) return CODA_OK;
  if (!q || !k || !v || !workspace) return CODA_EINVAL;
  const uintptr_t amask = is_half ? 7 : 15;    // four elements per load
  if ((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & amask) != 0 || ((ld_q | ld_k | ld_v) & 3) != 0) return CODA_EINVAL;
  if (ld_q < (long long)h * hd || ld_k < (long long)h * hd || ld_v < (long long)h * hd) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int bh = b * h;
  __nv_bfloat16 *qp = (__nv_bfloat16 *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  __nv_bfloat16 *kp = qp + (size_t)nsplit * bh * lq * hd;
  __nv_bfloat16 *vp = kp + (size_t)nsplit * bh * lk * hd;
  // q carries scale * log2(e): the kernel's softmax works in base 2.  All three tensors in one launch.
  PackJobs jobs = {};
  jobs.job[0] = {q, qp, lq, scale * LOG2E, ld_q};
  jobs.job[1] = {k, kp, lk, 1.0f, ld_k};
  jobs.job[2] = {v, vp, lk, 1.0f, ld_v};
  const long long t4 = (long long)(lq > lk ? lq : lk) * bh * hd / 4;
  const dim3 grid((unsigned)((t4 + 255) / 256), 3);
#define CODA_PACK(NS)                                                                 \
  if (is_half) pack_rows_multi_kernel<NS, true><<<grid, 256, 0, s>>>(jobs, b, h, hd); \
  else pack_rows_multi_kernel<NS, false><<<grid, 256, 0, s>>>(jobs, b, h, hd)
  if (nsplit == 1) { CODA_PACK(1); } else if (nsplit == 2) { CODA_PACK(2); } else { CODA_PACK(3); }
#undef CODA_PACK
  return launch_status();
}

int coda_attention_pack(int b, int h, int lq, int lk, int hd, int nsplit, float scale, const float *q,
                        const float *k, const float *v, void *workspace, void *stream) {
  const long long e = (long long)h * hd;
  return coda_attention_pack_strided(b, h, lq, lk, hd, nsplit, scale, q, k, v, e, e, e, 0, workspace, stream);
}

int coda_attention_fwd_packed(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                              float *out, float *lse, float dropout_p, unsigned int seed,
                              const unsigned int *seed_dev, void *stream) {
  return coda_attention_fwd_packed_ex(b, h, lq, lk, hd, nsplit, workspace, out, 0, lse, dropout_p, seed, seed_dev,
                                      stream);
}

int coda_attention_fwd_packed_ex(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                                 void *out_v, int out_half, float *lse, float dropout_p, unsigned int seed,
                                 const unsigned int *seed_dev, void *stream) {
  return coda_attention_fwd_packed_masked(b, h, lq, lk, hd, nsplit, workspace, out_v, out_half, lse, nullptr, dropout_p,
                                          seed, seed_dev, stream);
}

int coda_attention_fwd_packed_masked(int b, int h, int lq, int lk, int hd, int nsplit, const void *workspace,
                                     void *out_v, int out_half, float *lse, const unsigned long long *mask_q,
                                     float dropout_p, unsigned int seed, const unsigned int *seed_dev, void *stream) {
  float *out = reinterpret_cast<float *>(out_v);
  int st = attn_check(b, h, lq, lk, hd, nsplit);
  if (st != CODA_OK) return st;
  if (b == 0 || lq == 0) return CODA_OK;
  if (!out || !workspace || dropout_p < 0.f || dropout_p >= 1.f) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int bh = b * h;
  const __nv_bfloat16 *qp = (const __nv_bfloat16 *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  const __nv_bfloat16 *kp = qp + (size_t)nsplit * bh * lq * hd;
  const __nv_bfloat16 *vp = kp + (size_t)nsplit * bh * lk * hd;
  AttnMaps maps;
  for (int p = 0; p < nsplit; ++p) {
    st = make_tmap_k_major_16b(&maps.q[p], qp + (size_t)p * bh * lq * hd, 0, hd, lq, bh, hd, (long long)lq * hd, 64);
    if (st != CODA_OK) return st;
    st = make_tmap_k_major_16b(&maps.k[p], kp + (size_t)p * bh * lk * hd, 0, hd, lk, bh, hd, (long long)lk * hd, KT);
    if (st != CODA_OK) return st;
    st = make_tmap_k_major_16b(&maps.v[p], vp + (size_t)p * bh * lk * hd, 0, hd, lk, bh, hd, (long long)lk * hd, KT);
    if (st != CODA_OK) return st;
  }
  // fp16 output exists for the single key tile of the CLIP image tower (hd 64, nsplit <= 2, no mask)
  if (out_half && !(hd == 64 && lk <= KT && nsplit <= 2 && !mask_q)) return CODA_EINVAL;
#define CODA_ATTN(HD_, NS) \
  return launch_attn<HD_, NS>(maps, lq, lk, b, h, out, lse, dropout_p, seed, seed_dev, s, out_half, mask_q)
  if (hd == 64) {
    if (nsplit == 1) CODA_ATTN(64, 1);
    if (nsplit == 2) CODA_ATTN(64, 2);
    CODA_ATTN(64, 3);
  }
  if (nsplit == 1) CODA_ATTN(128, 1);
  if (nsplit == 2) CODA_ATTN(128, 2);
  CODA_ATTN(128, 3);
#undef CODA_ATTN
}

int coda_attention_fwd_half(int b, int h, int l, int hd, const void *q, const void *k, const void *v, long long ld_q,
                            long long ld_k, long long ld_v, void *out, void *workspace, void *stream) {
  // fp16 self-attention (the CLIP image tower, 12 x 64 heads).  At most one key tile (ViT-B/32: 50 tokens): q / k / v
  // are read as half (row-strided slices of the fused projection), re-laid as ONE plane of half operands -- fp16 is
  // the tensor core's native type, no bf16 split -- and the output is written as half.  Up to four key tiles
  // (ViT-B/16: 197 tokens): the resident kernel reads q / k / v by TMA in place, without a workspace.
  if (b < 0 || h <= 0 || l <= 0 || l > ResCfg::NT * KT || hd != 64 || (long long)b * h > 65535) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (l > KT) {
    if (!q || !k || !v || !out) return CODA_EINVAL;
    // TMA: 16-byte aligned bases and row strides
    if ((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) != 0 || ((ld_q | ld_k | ld_v) & 7) != 0) return CODA_EINVAL;
    if (ld_q < (long long)h * hd || ld_k < (long long)h * hd || ld_v < (long long)h * hd) return CODA_EINVAL;
    return launch_attn_half_resident(b, h, l, q, k, v, ld_q, ld_k, ld_v, reinterpret_cast<__half *>(out),
                                     (cudaStream_t)stream);
  }
  if (!q || !k || !v || !out || !workspace) return CODA_EINVAL;
  if ((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 7) != 0 || ((ld_q | ld_k | ld_v) & 3) != 0) return CODA_EINVAL;
  if (ld_q < (long long)h * hd || ld_k < (long long)h * hd || ld_v < (long long)h * hd) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int bh = b * h;
  __nv_bfloat16 *qp = (__nv_bfloat16 *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  __nv_bfloat16 *kp = qp + (size_t)bh * l * hd;
  __nv_bfloat16 *vp = kp + (size_t)bh * l * hd;
  PackJobs jobs = {};
  const float scale = 1.0f / sqrtf((float)hd);
  jobs.job[0] = {q, qp, l, scale * LOG2E, ld_q};
  jobs.job[1] = {k, kp, l, 1.0f, ld_k};
  jobs.job[2] = {v, vp, l, 1.0f, ld_v};
  const long long t4 = (long long)l * bh * hd / 4;
  pack_rows_half_kernel<<<dim3((unsigned)((t4 + 255) / 256), 3), 256, 0, s>>>(jobs, b, h, hd);
  int st = launch_status();
  if (st != CODA_OK) return st;
  AttnMaps maps;
  st = make_tmap_k_major_16b(&maps.q[0], qp, 1, hd, l, bh, hd, (long long)l * hd, 64);
  if (st != CODA_OK) return st;
  st = make_tmap_k_major_16b(&maps.k[0], kp, 1, hd, l, bh, hd, (long long)l * hd, KT);
  if (st != CODA_OK) return st;
  st = make_tmap_k_major_16b(&maps.v[0], vp, 1, hd, l, bh, hd, (long long)l * hd, KT);
  if (st != CODA_OK) return st;
  for (int p = 1; p < 3; ++p) { maps.q[p] = maps.q[0]; maps.k[p] = maps.k[0]; maps.v[p] = maps.v[0]; }
  return launch_attn<64, 1, true>(maps, l, l, b, h, reinterpret_cast<float *>(out), nullptr, 0.f, 0u, nullptr, s, 1);
}

int coda_attention_mask_pack(int b, int lq, int lk, const unsigned char *mask, long long stride_b, long long stride_q,
                             long long stride_k, unsigned long long *bits_q, unsigned long long *bits_k, void *stream) {
  if (b < 0 || lq <= 0 || lk <= 0) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!mask || !bits_q || !bits_k) return CODA_EINVAL;
  const long long nq = (long long)b * lq * ((lk + 63) / 64), nk = (long long)b * lk * ((lq + 63) / 64);
  cudaStream_t s = (cudaStream_t)stream;
  mask_pack_kernel<<<(unsigned)((nq + 127) / 128), 128, 0, s>>>(b, lq, lk, mask, stride_b, stride_q, stride_k, bits_q);
  mask_pack_kernel<<<(unsigned)((nk + 127) / 128), 128, 0, s>>>(b, lk, lq, mask, stride_b, stride_k, stride_q, bits_k);
  return launch_status();
}

int coda_attention_mask_radius(int b, int l, const float *xyz, float radius, unsigned long long *bits, void *stream) {
  if (b < 0 || l <= 0) return CODA_EINVAL;
  if (b == 0) return CODA_OK;
  if (!xyz || !bits) return CODA_EINVAL;
  const long long n = (long long)b * l * ((l + 63) / 64);
  mask_radius_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(b, l, xyz, radius, bits);
  return launch_status();
}

int coda_attention_dropout_mult(int bh, int lq, int lk, float dropout_p, unsigned int seed,
                                const unsigned int *seed_dev, float *mult, void *stream) {
  if (bh < 0 || lq < 0 || lk < 0 || dropout_p < 0.f || dropout_p >= 1.f) return CODA_EINVAL;
  const long long total = (long long)bh * lq * lk;
  if (total == 0) return CODA_OK;
  if (!mult) return CODA_EINVAL;
  dropout_mult_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      total, lq, lk, seed, seed_dev, drop_thresh32(dropout_p), 1.0f / (1.0f - dropout_p), mult);
  return launch_status();
}

int coda_attention_fwd(int b, int h, int lq, int lk, int hd, int nsplit, float scale, const float *q,
                       const float *k, const float *v, float *out, float *lse, float dropout_p,
                       unsigned int seed, const unsigned int *seed_dev, void *workspace, void *stream) {
  int st = coda_attention_pack(b, h, lq, lk, hd, nsplit, scale, q, k, v, workspace, stream);
  if (st != CODA_OK) return st;
  return coda_attention_fwd_packed(b, h, lq, lk, hd, nsplit, workspace, out, lse, dropout_p, seed, seed_dev, stream);
}

}  // extern "C"
