// Inference form of the pre-encoder's shared MLP + max over neighbours, ONE persistent kernel (sm_90a):
//
//     grouped rows (C0 = 3 | 6) --[C0 -> 64, fp32 FMAs]--> affine + ReLU --[64 -> 128, wgmma]--> affine + ReLU
//       --[128 -> 256, wgmma]--> affine + ReLU --> max over the 64 neighbours of each seed
//
// Each affine is an eval-mode BatchNorm folded on the host side: scale = gamma / sqrt(running_var + eps),
// shift = beta - running_mean * scale.  It is applied to every element BEFORE the max (gamma may be negative, so the
// max does not commute with it); the ReLU commutes with the max exactly (both are monotone), so it is applied once,
// to the pooled value.  No per-neighbour activation leaves the SM: HBM sees the grouped input once and the pooled
// output once.
//
// Layout:
//   * one consumer warpgroup per seed: the 64 rows of a seed are the M = 64 of the warpgroup's wgmmas.  Two
//     warpgroups per CTA work on different seeds, so that one's CUDA-core prologue / epilogue runs under the other's
//     tensor-core work.  Persistent CTAs, one per SM; seeds are dealt round-robin to the warpgroups.
//   * layer 1 is computed in exact fp32 straight into the register A fragments of layer 2 (each thread computes the
//     rows and columns its fragments hold), split into 3 bf16 planes in registers;
//   * layer 2's accumulator is mapped through affine + ReLU + the 3-plane split in registers and becomes layer 3's
//     register A operand (the m64nNk16 accumulator layout is the A-fragment layout, as for P.V in attention);
//   * layer 3 runs in two column halves of 128 (accumulator 64 registers + A fragments 96 registers per thread);
//     the max over rows is an in-thread max over the thread's two rows, an xor-shuffle over lane bits 2-4, and a
//     2 KB cross-warp step in shared memory.
//   * the weights are loaded ONCE per CTA by TMA and stay in shared memory: W2 on 3 bf16 planes (48 KB), W3 on the
//     first 2 planes of its 3-plane pack (128 KB; 3 planes would be 192 KB and, with W2, exceed the 227 KB a CTA can
//     have).  Plane products: 6 for layer 2, 5 for layer 3 (a1b1, a2b0, a1b0, a0b1, a0b0).
//   * no atomics: every output element is written by exactly one thread, in a fixed order of operations.
// C-ABI in include/coda_sa_mlp.h (coda_sa_mlp_max_infer).
#include "../../include/coda_sa_mlp.h"
#include "sm90_primitives.cuh"

using namespace coda;

namespace {

constexpr int GROUP = 64;                      // neighbours per seed = wgmma M
constexpr int C1 = 64, C2 = 128, C3 = 256;
constexpr int THREADS = 256;                   // two consumer warpgroups
constexpr int W2_PLANES = 3, W3_PLANES = 2;
constexpr int W2_TILE = C2 * 64 * 2;           // [128 rows][64 k] bf16, 128B-swizzled: 16 KB
constexpr int W3_TILE = C3 * 64 * 2;           // [256 rows][64 k] bf16 per 64-deep k-block: 32 KB
constexpr int W3_HALF = 128 * 128;             // byte offset of rows [128, 256) inside a W3 tile
constexpr int SMEM_W2 = W2_PLANES * W2_TILE;               // 48 KB
constexpr int SMEM_W3 = W3_PLANES * (C2 / 64) * W3_TILE;   // 128 KB
constexpr int AFFINE_FLOATS = 2 * (C1 + C2 + C3);          // scale1 shift1 scale2 shift2 scale3 shift3
constexpr int POOL_FLOATS = 2 * 2 * 4 * 128;               // [warpgroup][half][warp][128 columns]

// max(a, b) that returns NaN when either is NaN (fmaxf drops a NaN operand).  Every ReLU and the max over neighbours
// use it: the module path (relu, F.max_pool2d) carries a NaN through, so a non-finite neighbour makes NaN, not
// plausible features.  One FMNMX either way.
__device__ __forceinline__ float max_nan(float a, float b) {
  float d;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}

// layer-3 plane products (A plane, B plane), smallest terms first
__host__ __device__ constexpr int l3_a(int p) { return p == 0 ? 1 : p == 1 ? 2 : p == 2 ? 1 : 0; }
__host__ __device__ constexpr int l3_b(int p) { return p == 0 ? 1 : p == 1 ? 0 : p == 2 ? 0 : p == 3 ? 1 : 0; }

struct InferMaps {
  CUtensorMap w2[W2_PLANES];   // [128 rows][64 k] per plane, box [128][64]
  CUtensorMap w3[W3_PLANES];   // [256 rows][128 k] per plane, box [256][64]
};

struct InferParams {
  const float *x;              // grouped input (B, C0, npoint, 64), neighbour stride 1
  long long sx_b, sx_c, sx_p;  // element strides of batch, channel, seed
  int npoint;
  long long seeds;             // B * npoint
  const float *w1;             // (64, C0)
  const float *affine;         // AFFINE_FLOATS
  float *out;                  // (seeds, 256), row stride ldo
  long long ldo;
};

template <int C0>
__global__ void __launch_bounds__(THREADS, 1)
sa_infer_kernel(const __grid_constant__ InferMaps maps, const InferParams P) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char *smem = smem_align1024(smem_raw);
  unsigned char *w2s = smem;
  unsigned char *w3s = smem + SMEM_W2;                       // [plane][k-block] tiles
  float *w1s = reinterpret_cast<float *>(w3s + SMEM_W3);     // [C0][64]: a thread's column pair is one float2
  float *aff = w1s + C0 * C1;
  const float *s1 = aff, *h1 = aff + C1, *s2 = aff + 2 * C1, *h2 = s2 + C2, *s3 = h2 + C2, *h3 = s3 + C3;
  float *pool = aff + AFFINE_FLOATS;
  __shared__ __align__(8) uint64_t wbar;

  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(&wbar, 1);
    mbar_fence_init_cluster();
  }
  __syncthreads();
  if (tid == 0) {
#pragma unroll
    for (int p = 0; p < W2_PLANES; ++p) prefetch_tmap(&maps.w2[p]);
#pragma unroll
    for (int p = 0; p < W3_PLANES; ++p) prefetch_tmap(&maps.w3[p]);
    mbar_arrive_expect_tx(&wbar, (uint32_t)(SMEM_W2 + SMEM_W3));
#pragma unroll
    for (int p = 0; p < W2_PLANES; ++p) tma_load_3d(w2s + p * W2_TILE, &maps.w2[p], &wbar, 0, 0, 0);
#pragma unroll
    for (int p = 0; p < W3_PLANES; ++p)
#pragma unroll
      for (int kb = 0; kb < C2 / 64; ++kb)
        tma_load_3d(w3s + (p * (C2 / 64) + kb) * W3_TILE, &maps.w3[p], &wbar, kb * 64, 0, 0);
  }
  for (int i = tid; i < C0 * C1; i += THREADS) {
    const int c = i / C1, o = i % C1;
    w1s[i] = __ldg(P.w1 + o * C0 + c);
  }
  for (int i = tid; i < AFFINE_FLOATS; i += THREADS) aff[i] = __ldg(P.affine + i);
  __syncthreads();
  mbar_wait(&wbar, 0);

  const int wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int r0 = warp * 16 + g;                              // this thread's rows r0, r0 + 8 of the seed
  float *mypool = pool + wg * (2 * 4 * 128);
  const long long step = (long long)gridDim.x * 2;
  long long s = (long long)blockIdx.x * 2 + wg;

  // grouped input of a seed: the thread's two rows of every channel
  float xin[C0][2];
  auto load_x = [&](long long seed) {
    const long long b = seed / P.npoint, p = seed - b * P.npoint;
    const float *xs = P.x + b * P.sx_b + p * P.sx_p;
#pragma unroll
    for (int c = 0; c < C0; ++c) {
      xin[c][0] = __ldg(xs + c * P.sx_c + r0);
      xin[c][1] = __ldg(xs + c * P.sx_c + r0 + 8);
    }
  };
  if (s < P.seeds) load_x(s);

  for (; s < P.seeds; s += step) {
    // ---- layer 1 (fp32 FMAs) -> affine + ReLU -> 3 bf16 planes = register A of layer 2.  Register q of k-step kk
    // holds (row r0 + 8 (q & 1), columns 16 kk + 8 (q >> 1) + 2 t4 + {0, 1}).
    uint32_t a2f[C1 / 16][3][4];
#pragma unroll
    for (int kk = 0; kk < C1 / 16; ++kk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = q & 1, col = kk * 16 + (q >> 1) * 8 + 2 * t4;
        float v0 = 0.f, v1 = 0.f;
#pragma unroll
        for (int c = 0; c < C0; ++c) {
          const float2 w = *reinterpret_cast<const float2 *>(w1s + c * C1 + col);
          v0 = fmaf(w.x, xin[c][i], v0);
          v1 = fmaf(w.y, xin[c][i], v1);
        }
        v0 = max_nan(fmaf(v0, s1[col], h1[col]), 0.f);
        v1 = max_nan(fmaf(v1, s1[col + 1], h1[col + 1]), 0.f);
        uint32_t w[3];
        split_pair<3>(v0, v1, w);
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) a2f[kk][pl][q] = w[pl];
      }
    }
    // the next seed's input is in flight during this seed's tensor-core work
    if (s + step < P.seeds) load_x(s + step);

    // ---- layer 2: 64 x 128 x 64, the six plane products of 3 x 3 planes
    float acc2[C2 / 2];
    acc_fence(acc2);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < n_products(3); ++p) {
      const uint64_t bd = gmma_desc_k_sw128(w2s + prod_b(3, p) * W2_TILE);
#pragma unroll
      for (int kk = 0; kk < C1 / 16; ++kk)
        Wgmma<128, false>::template rs<0>(acc2, a2f[kk][prod_a(3, p)], gmma_desc_advance(bd, kk * 32), (p | kk) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc2);

    // ---- layer 2 epilogue: affine + ReLU + 3-plane split; accumulator chunk c (columns 8c..8c+7) feeds register
    // q >> 1 of k-step c / 2 of layer 3
    uint32_t a3f[C2 / 16][3][4];
#pragma unroll
    for (int kk = 0; kk < C2 / 16; ++kk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = q & 1, c = 2 * kk + (q >> 1), col = c * 8 + 2 * t4;
        const float v0 = max_nan(fmaf(acc2[c * 4 + i * 2], s2[col], h2[col]), 0.f);
        const float v1 = max_nan(fmaf(acc2[c * 4 + i * 2 + 1], s2[col + 1], h2[col + 1]), 0.f);
        uint32_t w[3];
        split_pair<3>(v0, v1, w);
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) a3f[kk][pl][q] = w[pl];
      }
    }

    // ---- layer 3 in two column halves: 64 x 128 x 128 each, five plane products -> affine -> max -> ReLU
    float *orow = P.out + s * P.ldo;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float acc3[64];
      acc_fence(acc3);
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < 5; ++p) {
#pragma unroll
        for (int kk = 0; kk < C2 / 16; ++kk) {
          const unsigned char *bt = w3s + (l3_b(p) * (C2 / 64) + kk / 4) * W3_TILE + h * W3_HALF;
          Wgmma<128, false>::template rs<0>(acc3, a3f[kk][l3_a(p)], gmma_desc_advance(gmma_desc_k_sw128(bt), (kk & 3) * 32),
                                            (p | kk) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc3);
      float *buf = mypool + h * (4 * 128);
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const int col = h * 128 + c * 8 + 2 * t4;
        const float sc0 = s3[col], sh0 = h3[col], sc1 = s3[col + 1], sh1 = h3[col + 1];
        float m0 = max_nan(fmaf(acc3[c * 4], sc0, sh0), fmaf(acc3[c * 4 + 2], sc0, sh0));
        float m1 = max_nan(fmaf(acc3[c * 4 + 1], sc1, sh1), fmaf(acc3[c * 4 + 3], sc1, sh1));
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {       // the warp's 16 rows: lane bits 2..4
          m0 = max_nan(m0, __shfl_xor_sync(0xffffffffu, m0, o));
          m1 = max_nan(m1, __shfl_xor_sync(0xffffffffu, m1, o));
        }
        if (g == 0) *reinterpret_cast<float2 *>(buf + warp * 128 + c * 8 + 2 * t4) = make_float2(m0, m1);
      }
      // the four warps' maxima -> one column per thread.  Buffers alternate with h: a buffer is rewritten one seed
      // later, after the barrier of the other half, which every thread reaches only after reading it.
      bar_sync(1 + wg, 128);
      const int tl = tid & 127;
      const float m = max_nan(max_nan(buf[tl], buf[128 + tl]), max_nan(buf[256 + tl], buf[384 + tl]));
      orow[h * 128 + tl] = max_nan(m, 0.f);
    }
  }
}

template <int C0>
int launch_infer(const InferMaps &maps, const InferParams &P, cudaStream_t s) {
  constexpr size_t smem = 1024 + SMEM_W2 + SMEM_W3 + (size_t)(C0 * C1 + AFFINE_FLOATS + POOL_FLOATS) * 4;
  static_assert(smem <= 227 * 1024 - 1024, "shared memory");
  constexpr auto kern = sa_infer_kernel<C0>;
  if (const int st = raise_smem_limit<kern>((int)smem)) return st;
  const long long pairs = (P.seeds + 1) / 2;
  const unsigned grid = (unsigned)(pairs < sm_count() ? pairs : sm_count());
  kern<<<grid, THREADS, smem, s>>>(maps, P);
  return launch_status();
}

}  // namespace

extern "C" {

int coda_sa_mlp_max_infer(long long batch, int c0, int npoint, int nsample, const float *x, long long x_batch_stride,
                          long long x_channel_stride, long long x_point_stride, const float *w1, const void *w2_planes,
                          long long w2_plane_stride, const void *w3_planes, long long w3_plane_stride,
                          const float *affine, float *out, long long ldo, void *stream) {
  if (batch < 0 || npoint < 0 || (c0 != 3 && c0 != 6) || nsample != GROUP) return CODA_EINVAL;
  if (batch == 0 || npoint == 0) return CODA_OK;
  if (!x || !w1 || !w2_planes || !w3_planes || !affine || !out || ldo < C3) return CODA_EINVAL;
  if (((uintptr_t)w2_planes & 15) || ((uintptr_t)w3_planes & 15) || (w2_plane_stride & 7) || (w3_plane_stride & 7))
    return CODA_EINVAL;                                      // TMA: 16-byte aligned plane bases
  InferMaps maps;
  const char *b2 = (const char *)w2_planes, *b3 = (const char *)w3_planes;
  for (int p = 0; p < W2_PLANES; ++p) {
    const int st = make_tmap_k_major_16b(&maps.w2[p], b2 + (size_t)p * w2_plane_stride * 2, 0, C1, C2, 1, C1, 0, C2);
    if (st != CODA_OK) return st;
  }
  for (int p = 0; p < W3_PLANES; ++p) {
    const int st = make_tmap_k_major_16b(&maps.w3[p], b3 + (size_t)p * w3_plane_stride * 2, 0, C2, C3, 1, C2, 0, C3);
    if (st != CODA_OK) return st;
  }
  InferParams P;
  P.x = x; P.sx_b = x_batch_stride; P.sx_c = x_channel_stride; P.sx_p = x_point_stride;
  P.npoint = npoint; P.seeds = batch * npoint; P.w1 = w1; P.affine = affine; P.out = out; P.ldo = ldo;
  cudaStream_t s = (cudaStream_t)stream;
  return c0 == 3 ? launch_infer<3>(maps, P, s) : launch_infer<6>(maps, P, s);
}

}  // extern "C"
