// PointNet++ set-abstraction ops for H100 (sm_90a) behind the C-ABI declared
// in include/coda_pointnet2.h.  Written from the behaviour of the reference's
// `pointnet2._ext` (third_party_pointnet2/pointnet2/_ext_src/src/*.cu), not
// from its code: the reference runs one CTA per scene and one thread per ball
// centre; here FPS is a thread-block-cluster kernel that keeps the whole scene
// in registers and exchanges one 32-byte record per round over DSMEM, and
// ball-query / three-nn are tiled through shared memory with warp ballots.
#include <math.h>

#include "../../include/coda_pointnet2.h"
#include "coda_common.cuh"

using namespace coda;

namespace {

// =====================================================================
//  Furthest point sampling
// =====================================================================
//
// Reference semantics (sampling_gpu.cu:72-176), restated:
//   * temp[k] = 1e10, idx[0] = 0, old = 0
//   * each round: for every k with |p_k|^2 > 1e-3:  temp[k] = min(temp[k], |p_k - p_old|^2);
//     old = argmax temp[k];  ties are resolved by the reference's thread layout:
//     thread t owns k = t (mod bs) and keeps its smallest k; the halving tree
//     keeps the lower slot on ties at every level, so the last level (slot 0
//     vs 1) is decided by bit 0 of t, the one before by bit 1, ...  =>  the
//     winner among equal maxima is the lexicographic minimum of
//     (bitrev_{log2 bs}(k mod bs), k div bs).
//   * if no point is valid the tree yields (best = -1, idx 0).
//
// This kernel works in "position space":  p = bitrev(k mod bs) * R + k div bs
// with R = ceil(n / bs), so the tie rule becomes "smallest p wins".  Positions
// are dealt round-robin to the CL*512 threads of a cluster (CL CTAs per scene),
// each thread keeps PPT positions (x, y, z, temp) in registers for the whole
// kernel.  A round is: PPT distance updates per thread -> two redux.sync per
// warp (max of value bits, min of position) -> one __syncthreads -> every
// warp re-reduces the 16 warp records -> (CL > 1) each CTA pushes its 32-byte
// record into every peer's shared memory with st.async + mbarrier complete_tx
// and waits on its own mbarrier -> every thread knows the winner and its
// coordinates.  No global memory is read after the prologue.

constexpr int FPS_T = 512;
constexpr int FPS_WARPS = FPS_T / 32;
constexpr int FPS_MAX_CL = 8;
constexpr int FPS_MAX_PPT = 16;
constexpr int INT_BIG = 0x7fffffff;

struct __align__(16) FpsRec {  // 32 bytes, exchanged between CTAs
  int m;                       // value bits of the CTA's best temp (>= 0), or < 0: none
  int p;                       // position of that point
  int k;                       // its index in the scene
  int pad;
  float x, y, z, w;
};

struct FpsSmem {
  FpsRec crec[2][FPS_MAX_CL];
  uint64_t mbar[2];
  int2 wrec[2][FPS_WARPS];
};

template <int PPT>
__global__ void __launch_bounds__(FPS_T, 1)
fps_cluster_kernel(int n, int m, int bs_log2, int R, int cl_log2,
                   const float *__restrict__ xyz, int *__restrict__ idx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FpsSmem &sm = *reinterpret_cast<FpsSmem *>(smem_raw);
  float4 *spts = reinterpret_cast<float4 *>(smem_raw + sizeof(FpsSmem));

  const int CL = 1 << cl_log2;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int rank = (cl_log2 > 0) ? (int)cluster_ctarank() : 0;
  const int scene = blockIdx.x >> cl_log2;
  const int gt_log2 = cl_log2 + 9;       // log2(CL * FPS_T)
  const int g = (rank << 9) + tid;       // thread id within the scene's cluster
  const int P = R << bs_log2;

  xyz += (size_t)scene * n * 3;
  idx += (size_t)scene * m;

  // ---- prologue: load my positions -------------------------------------
  float px[PPT], py[PPT], pz[PPT], pt[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) {
    const int p = g + (i << gt_log2);
    const int c = p / R, r = p - c * R;
    const int cb = bs_log2 ? (int)(__brev((unsigned)c) >> (32 - bs_log2)) : 0;
    const int k = cb + (r << bs_log2);
    bool valid = (p < P) && (k < n);
    float x = 0.f, y = 0.f, z = 0.f;
    if (valid) {
      x = __ldg(xyz + (size_t)k * 3 + 0);
      y = __ldg(xyz + (size_t)k * 3 + 1);
      z = __ldg(xyz + (size_t)k * 3 + 2);
      // sampling_gpu.cu:103-104 (mag compared against the double constant 1e-3)
      const float mag = __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
      valid = !((double)mag <= 1e-3);
    }
    px[i] = x; py[i] = y; pz[i] = z;
    pt[i] = valid ? 1e10f : -1.0f;  // -1 never beats `best` (strict >)
    spts[(i << 9) + tid] = make_float4(x, y, z, __int_as_float(valid ? k : 0));
  }
  // first sample is always point 0 (sampling_gpu.cu:88-89)
  const float p0x = __ldg(xyz + 0), p0y = __ldg(xyz + 1), p0z = __ldg(xyz + 2);
  float cx = p0x, cy = p0y, cz = p0z;
  if (rank == 0 && tid == 0) idx[0] = 0;

  if (cl_log2 > 0) {
    if (tid == 0) {
      mbar_init(&sm.mbar[0], 1);
      mbar_init(&sm.mbar[1], 1);
      mbar_fence_init_cluster();
      mbar_arrive_expect_tx(&sm.mbar[0], (uint32_t)(CL * sizeof(FpsRec)));
      mbar_arrive_expect_tx(&sm.mbar[1], (uint32_t)(CL * sizeof(FpsRec)));
    }
    cluster_sync_all();  // barriers initialised and armed before any peer store
  } else {
    __syncthreads();
  }

  for (int j = 1; j < m; ++j) {
    const int buf = j & 1;
    // ---- per-thread update (sampling_gpu.cu:100-113) ---------------------
    float best = -1.0f;
    int bi = 0;
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
      const float dx = __fsub_rn(px[i], cx), dy = __fsub_rn(py[i], cy),
                  dz = __fsub_rn(pz[i], cz);
      const float d =
          __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
      const float t = fminf(d, pt[i]);
      pt[i] = t;
      if (t > best) { best = t; bi = i; }  // ascending position => smallest p kept
    }
    // ---- warp argmax: max value bits, then min position -------------------
    const int mb = __float_as_int(best);
    const int pos = g + (bi << gt_log2);
    const int wm = __reduce_max_sync(0xffffffffu, mb);
    const unsigned cand = (mb == wm) ? (unsigned)pos : (unsigned)INT_BIG;
    const unsigned wp = __reduce_min_sync(0xffffffffu, cand);
    if (cand == wp) sm.wrec[buf][warp] = make_int2(wm, (int)wp);
    __syncthreads();
    // ---- CTA argmax (every warp redundantly; no second barrier) ----------
    int2 r2 = (lane < FPS_WARPS) ? sm.wrec[buf][lane] : make_int2(INT_MIN, INT_BIG);
    const int M = __reduce_max_sync(0xffffffffu, r2.x);
    const unsigned c2 = (r2.x == M) ? (unsigned)r2.y : (unsigned)INT_BIG;
    const int Pm = (int)__reduce_min_sync(0xffffffffu, c2);
    // local slot of position Pm in this CTA's spts
    const int slot = ((Pm >> gt_log2) << 9) + ((Pm & ((1 << gt_log2) - 1)) - (rank << 9));
    int win_k;
    float wx, wy, wz;
    if (cl_log2 == 0) {
      if (M >= 0) {
        const float4 w = spts[slot];
        wx = w.x; wy = w.y; wz = w.z; win_k = __float_as_int(w.w);
      } else {  // no valid point at all: reference tree returns index 0
        wx = p0x; wy = p0y; wz = p0z; win_k = 0;
      }
    } else {
      // ---- cluster exchange: push my record to every CTA of the cluster ---
      if (warp == 0 && lane < CL) {
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (M >= 0) w = spts[slot];
        const uint32_t dst = mapa_u32(smem_u32(&sm.crec[buf][rank]), (uint32_t)lane);
        const uint32_t bar = mapa_u32(smem_u32(&sm.mbar[buf]), (uint32_t)lane);
        st_async_v4(dst, bar, (uint32_t)M, (uint32_t)Pm, __float_as_uint(w.w), 0u);
        st_async_v4(dst + 16, bar, __float_as_uint(w.x), __float_as_uint(w.y),
                    __float_as_uint(w.z), 0u);
      }
      mbar_wait(&sm.mbar[buf], (uint32_t)(((j - 1) >> 1) & 1));  // u-th use of this buffer
      int rm = INT_MIN, rp = INT_BIG;
      if (lane < CL) { rm = sm.crec[buf][lane].m; rp = sm.crec[buf][lane].p; }
      const int Mg = __reduce_max_sync(0xffffffffu, rm);
      const unsigned c3 = (rm == Mg) ? (unsigned)rp : (unsigned)INT_BIG;
      const unsigned Pg = __reduce_min_sync(0xffffffffu, c3);
      const unsigned owner_mask = __ballot_sync(0xffffffffu, lane < CL && c3 == Pg);
      const int owner = __ffs(owner_mask) - 1;
      if (Mg >= 0) {
        const FpsRec &w = sm.crec[buf][owner];
        wx = w.x; wy = w.y; wz = w.z; win_k = w.k;
      } else {
        wx = p0x; wy = p0y; wz = p0z; win_k = 0;
      }
      // every thread of this CTA has consumed crec[buf] only after the NEXT
      // __syncthreads; re-arm the barrier for round j+2 now (tx-count may be
      // armed before or after peers' complete_tx, both are legal).
      if (tid == 0 && j + 2 < m)
        mbar_arrive_expect_tx(&sm.mbar[buf], (uint32_t)(CL * sizeof(FpsRec)));
    }
    cx = wx; cy = wy; cz = wz;
    if (rank == 0 && tid == 0) idx[j] = win_k;
  }
  if (cl_log2 > 0) cluster_sync_all();  // no CTA exits while peers may still store to it
}

// Fallback for scenes too large for the register-resident kernel: one CTA per
// scene, temp in global scratch, same key (value bits, then smallest position).
__global__ void __launch_bounds__(1024, 1)
fps_generic_kernel(int n, int m, int bs_log2, int R, const float *__restrict__ xyz,
                   float *__restrict__ temp, int *__restrict__ idx) {
  __shared__ int2 wrec[2][32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int scene = blockIdx.x;
  xyz += (size_t)scene * n * 3;
  temp += (size_t)scene * n;
  idx += (size_t)scene * m;
  const int bs_mask = (1 << bs_log2) - 1;
  for (int k = tid; k < n; k += 1024) {
    const float x = xyz[k * 3], y = xyz[k * 3 + 1], z = xyz[k * 3 + 2];
    const float mag = __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
    temp[k] = ((double)mag <= 1e-3) ? -1.0f : 1e10f;
  }
  if (tid == 0) idx[0] = 0;
  int old = 0;
  __syncthreads();
  for (int j = 1; j < m; ++j) {
    const int buf = j & 1;
    const float cx = xyz[old * 3], cy = xyz[old * 3 + 1], cz = xyz[old * 3 + 2];
    int mb = __float_as_int(-1.0f);
    unsigned bp = (unsigned)INT_BIG;
    for (int k = tid; k < n; k += 1024) {
      float t = temp[k];
      if (t >= 0.f) {
        const float dx = __fsub_rn(xyz[k * 3], cx), dy = __fsub_rn(xyz[k * 3 + 1], cy),
                    dz = __fsub_rn(xyz[k * 3 + 2], cz);
        const float d = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
        t = fminf(d, t);
        temp[k] = t;
        const int c = k & bs_mask;
        const int cb = bs_log2 ? (int)(__brev((unsigned)c) >> (32 - bs_log2)) : 0;
        const unsigned p = (unsigned)(cb * R + (k >> bs_log2));
        const int tb = __float_as_int(t);
        if (tb > mb || (tb == mb && p < bp)) { mb = tb; bp = p; }
      }
    }
    const int wm = __reduce_max_sync(0xffffffffu, mb);
    const unsigned cand = (mb == wm) ? bp : (unsigned)INT_BIG;
    const unsigned wp = __reduce_min_sync(0xffffffffu, cand);
    if (lane == 0) wrec[buf][warp] = make_int2(wm, (int)wp);
    __syncthreads();
    const int2 r2 = wrec[buf][lane];
    const int M = __reduce_max_sync(0xffffffffu, r2.x);
    const unsigned c2 = (r2.x == M) ? (unsigned)r2.y : (unsigned)INT_BIG;
    const unsigned Pm = __reduce_min_sync(0xffffffffu, c2);
    if (M >= 0) {
      const int c = (int)(Pm / (unsigned)R), r = (int)(Pm - (unsigned)c * R);
      const int cb = bs_log2 ? (int)(__brev((unsigned)c) >> (32 - bs_log2)) : 0;
      old = cb + (r << bs_log2);
    } else {
      old = 0;
    }
    if (tid == 0) idx[j] = old;
  }
}

int g_fps_force_cluster = 0;

// include/cuda_utils.h:17-21 of the reference: the block size its launcher
// picks, which defines the tie rule.  Same double-precision expression.
inline int ref_block_size_log2(int n) {
  int pow_2 = (int)(log((double)n) / log(2.0));
  int t = 1 << pow_2;
  if (t > 512) pow_2 = 9;
  if (t < 1) pow_2 = 0;
  return pow_2;
}

template <int PPT>
int launch_fps(int b, int n, int m, int bs_log2, int R, int cl_log2,
               const float *xyz, int *idx, cudaStream_t s) {
  const size_t smem = sizeof(FpsSmem) + (size_t)PPT * FPS_T * sizeof(float4);
  cudaError_t e = cudaFuncSetAttribute(fps_cluster_kernel<PPT>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  if (e != cudaSuccess) return (int)e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(b << cl_log2));
  cfg.blockDim = dim3(FPS_T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1u << cl_log2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, fps_cluster_kernel<PPT>, n, m, bs_log2, R, cl_log2,
                         xyz, idx);
  return e == cudaSuccess ? CODA_OK : (int)e;
}

// =====================================================================
//  ball query (+ fused grouping of xyz)
// =====================================================================
// One warp per ball centre; the scene streams through shared memory in tiles
// that all 8 warps of the CTA share; each lane tests one point per step and a
// ballot + popc prefix keeps the hits in ascending index order, which is the
// reference's "first nsample in scan order" rule (ball_query_gpu.cu:25-45).
constexpr int BQ_WARPS = 8;
constexpr int BQ_T = BQ_WARPS * 32;
constexpr int BQ_TILE = 2048;  // points per tile (24 KB)

template <bool GROUP>
__global__ void __launch_bounds__(BQ_T)
ball_query_kernel(int n, int m, float radius2, int nsample, int normalize,
                  float inv_radius, const float *__restrict__ xyz,
                  const float *__restrict__ new_xyz, int *__restrict__ idx,
                  float *__restrict__ grouped) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float *tile = reinterpret_cast<float *>(smem_raw);                   // BQ_TILE*3
  int *hits = reinterpret_cast<int *>(smem_raw + BQ_TILE * 3 * sizeof(float));  // BQ_WARPS*nsample
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  const int j = blockIdx.x * BQ_WARPS + warp;
  const bool active = j < m;
  xyz += (size_t)b * n * 3;
  int *myhits = hits + warp * nsample;

  float cxv = 0.f, cyv = 0.f, czv = 0.f;
  if (active) {
    const float *c = new_xyz + ((size_t)b * m + j) * 3;
    cxv = __ldg(c); cyv = __ldg(c + 1); czv = __ldg(c + 2);
  }
  int cnt = active ? 0 : nsample;  // inactive warps count as finished

  for (int base = 0; base < n; base += BQ_TILE) {
    const int tn = min(BQ_TILE, n - base);
    const float *src = xyz + (size_t)base * 3;
    for (int i = tid; i < tn * 3; i += BQ_T) tile[i] = __ldg(src + i);
    __syncthreads();
    if (cnt < nsample) {
      for (int kk = 0; kk < tn; kk += 32) {
        const int k = kk + lane;
        bool hit = false;
        if (k < tn) {
          const float x = tile[k * 3], y = tile[k * 3 + 1], z = tile[k * 3 + 2];
          // ball_query_gpu.cu:34-35: (new_x - x)^2 + ... -> FMUL(dy,dy), FFMA(dx,dx,.), FFMA(dz,dz,.) (reference SASS)
          const float dx = __fsub_rn(cxv, x), dy = __fsub_rn(cyv, y), dz = __fsub_rn(czv, z);
          const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
          hit = d2 < radius2;
        }
        const unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (mask) {
          const int slot = cnt + __popc(mask & ((1u << lane) - 1u));
          if (hit && slot < nsample) myhits[slot] = base + k;
          cnt += __popc(mask);
          if (cnt >= nsample) break;
        }
      }
    }
    // all warps done -> stop streaming; doubles as the barrier before the
    // next tile overwrites shared memory
    if (__syncthreads_and(cnt >= nsample)) break;
  }
  if (!active) return;
  __syncwarp();
  const int got = min(cnt, nsample);
  const int first = got > 0 ? myhits[0] : 0;  // ball_query_gpu.cu:37-41 / zeros
  int *orow = idx + ((size_t)b * m + j) * nsample;
  for (int s = lane; s < nsample; s += 32) {
    const int k = s < got ? myhits[s] : first;
    orow[s] = k;
    if (GROUP) {
      // pointnet2_utils.py:346-349: group xyz^T, "-= new_xyz", "/= radius"
      // (torch's CUDA division by a scalar multiplies by the fp32 reciprocal)
      const float *p = xyz + (size_t)k * 3;
      float vx = __fsub_rn(__ldg(p), cxv), vy = __fsub_rn(__ldg(p + 1), cyv),
            vz = __fsub_rn(__ldg(p + 2), czv);
      if (normalize) {
        vx = __fmul_rn(vx, inv_radius); vy = __fmul_rn(vy, inv_radius);
        vz = __fmul_rn(vz, inv_radius);
      }
      const size_t ms = (size_t)m * nsample;
      float *g = grouped + (size_t)b * 3 * ms + (size_t)j * nsample + s;
      g[0] = vx; g[ms] = vy; g[2 * ms] = vz;
    }
  }
}

// =====================================================================
//  gather / group (+ grads), three_nn, three_interpolate (+ grad)
// =====================================================================
__global__ void gather_points_kernel(int c, int n, int m,
                                     const float *__restrict__ points,
                                     const int *__restrict__ idx,
                                     float *__restrict__ out) {
  const int b = blockIdx.z, l = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int a = __ldg(idx + (size_t)b * m + j);
  out[((size_t)b * c + l) * m + j] = __ldg(points + ((size_t)b * c + l) * n + a);
}

__global__ void gather_points_grad_kernel(int c, int n, int m,
                                          const float *__restrict__ grad_out,
                                          const int *__restrict__ idx,
                                          float *__restrict__ grad_points) {
  const int b = blockIdx.z, l = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int a = __ldg(idx + (size_t)b * m + j);
  atomicAdd(grad_points + ((size_t)b * c + l) * n + a,
            __ldg(grad_out + ((size_t)b * c + l) * m + j));
}

// thread per (j, s) element; channels are split over blockIdx.y so that small-c
// launches still fill the machine; writes are coalesced along (j, s).
__global__ void group_points_kernel(int c, int n, int ms, int c_per_block,
                                    const float *__restrict__ points,
                                    const int *__restrict__ idx,
                                    float *__restrict__ out) {
  const int b = blockIdx.z;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ms) return;
  const int ii = __ldg(idx + (size_t)b * ms + e);
  const int l0 = blockIdx.y * c_per_block, l1 = min(c, l0 + c_per_block);
  for (int l = l0; l < l1; ++l)
    out[((size_t)b * c + l) * ms + e] = __ldg(points + ((size_t)b * c + l) * n + ii);
}

__global__ void group_points_grad_kernel(int c, int n, int ms, int c_per_block,
                                         const float *__restrict__ grad_out,
                                         const int *__restrict__ idx,
                                         float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ms) return;
  const int ii = __ldg(idx + (size_t)b * ms + e);
  const int l0 = blockIdx.y * c_per_block, l1 = min(c, l0 + c_per_block);
  for (int l = l0; l < l1; ++l)
    atomicAdd(grad_points + ((size_t)b * c + l) * n + ii,
              __ldg(grad_out + ((size_t)b * c + l) * ms + e));
}

constexpr int NN_T = 256;
constexpr int NN_TILE = 1024;
// thread per unknown point; known points stream through shared memory and are
// read as warp broadcasts.  The reference's double-typed bests hold fp32 values
// (or 1e40 == +inf after the float cast), so fp32 bests initialised to +inf
// with strict < are equivalent (interpolate_gpu.cu:30-53).
__global__ void __launch_bounds__(NN_T)
three_nn_kernel(int n, int m, const float *__restrict__ unknown,
                const float *__restrict__ known, float *__restrict__ dist2,
                int *__restrict__ idx) {
  __shared__ float tile[NN_TILE * 3];
  const int b = blockIdx.y;
  const int j = blockIdx.x * NN_T + threadIdx.x;
  known += (size_t)b * m * 3;
  float ux = 0.f, uy = 0.f, uz = 0.f;
  if (j < n) {
    const float *u = unknown + ((size_t)b * n + j) * 3;
    ux = __ldg(u); uy = __ldg(u + 1); uz = __ldg(u + 2);
  }
  float b1 = INFINITY, b2 = INFINITY, b3 = INFINITY;
  int i1 = 0, i2 = 0, i3 = 0;
  for (int base = 0; base < m; base += NN_TILE) {
    const int tn = min(NN_TILE, m - base);
    __syncthreads();
    for (int i = threadIdx.x; i < tn * 3; i += NN_T) tile[i] = __ldg(known + (size_t)base * 3 + i);
    __syncthreads();
    for (int k = 0; k < tn; ++k) {
      const float dx = __fsub_rn(ux, tile[k * 3]), dy = __fsub_rn(uy, tile[k * 3 + 1]),
                  dz = __fsub_rn(uz, tile[k * 3 + 2]);
      const float d = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
      const int kk = base + k;
      if (d < b1) {
        b3 = b2; i3 = i2; b2 = b1; i2 = i1; b1 = d; i1 = kk;
      } else if (d < b2) {
        b3 = b2; i3 = i2; b2 = d; i2 = kk;
      } else if (d < b3) {
        b3 = d; i3 = kk;
      }
    }
  }
  if (j < n) {
    float *D = dist2 + ((size_t)b * n + j) * 3;
    int *I = idx + ((size_t)b * n + j) * 3;
    D[0] = b1; D[1] = b2; D[2] = b3;
    I[0] = i1; I[1] = i2; I[2] = i3;
  }
}

__global__ void three_interpolate_kernel(int c, int m, int n, int c_per_block,
                                         const float *__restrict__ points,
                                         const int *__restrict__ idx,
                                         const float *__restrict__ weight,
                                         float *__restrict__ out) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float *w = weight + ((size_t)b * n + j) * 3;
  const int *ii = idx + ((size_t)b * n + j) * 3;
  const float w1 = __ldg(w), w2 = __ldg(w + 1), w3 = __ldg(w + 2);
  const int i1 = __ldg(ii), i2 = __ldg(ii + 1), i3 = __ldg(ii + 2);
  const int l0 = blockIdx.y * c_per_block, l1 = min(c, l0 + c_per_block);
  for (int l = l0; l < l1; ++l) {
    const float *p = points + ((size_t)b * c + l) * m;
    // interpolate_gpu.cu:101-102: p1*w1 + p2*w2 + p3*w3 -> FMUL(p2,w2), FFMA(p1,w1), FFMA(p3,w3)
    out[((size_t)b * c + l) * n + j] =
        __fmaf_rn(__ldg(p + i3), w3, __fmaf_rn(__ldg(p + i1), w1, __fmul_rn(__ldg(p + i2), w2)));
  }
}

__global__ void three_interpolate_grad_kernel(int c, int n, int m, int c_per_block,
                                              const float *__restrict__ grad_out,
                                              const int *__restrict__ idx,
                                              const float *__restrict__ weight,
                                              float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float *w = weight + ((size_t)b * n + j) * 3;
  const int *ii = idx + ((size_t)b * n + j) * 3;
  const float w1 = __ldg(w), w2 = __ldg(w + 1), w3 = __ldg(w + 2);
  const int i1 = __ldg(ii), i2 = __ldg(ii + 1), i3 = __ldg(ii + 2);
  const int l0 = blockIdx.y * c_per_block, l1 = min(c, l0 + c_per_block);
  for (int l = l0; l < l1; ++l) {
    const float go = __ldg(grad_out + ((size_t)b * c + l) * n + j);
    float *g = grad_points + ((size_t)b * c + l) * m;
    atomicAdd(g + i1, __fmul_rn(go, w1));
    atomicAdd(g + i2, __fmul_rn(go, w2));
    atomicAdd(g + i3, __fmul_rn(go, w3));
  }
}

inline int pick_c_per_block(int c, long long work_items_per_channel, int b) {
  // aim for >= ~4 waves of 132 SMs worth of 256-thread CTAs, at least 1 channel
  const long long ctas_per_channel_slice = (work_items_per_channel + 255) / 256 * b;
  int slices = (int)((132LL * 8 + ctas_per_channel_slice - 1) / ctas_per_channel_slice);
  if (slices < 1) slices = 1;
  if (slices > c) slices = c;
  return (c + slices - 1) / slices;
}

}  // namespace

// =====================================================================
//  C-ABI
// =====================================================================
extern "C" {

int coda_abi_version(void) { return 1; }

const char *coda_status_string(int status) {
  if (status == CODA_OK) return "ok";
  if (status == CODA_EINVAL) return "coda: invalid argument (shape or null pointer)";
  if (status == CODA_ETOOLARGE) return "coda: problem too large for this entry point";
  return cudaGetErrorString((cudaError_t)status);
}

int coda_fps_set_cluster(int cluster_ctas) {
  const int old = g_fps_force_cluster;
  if (cluster_ctas == 0 || cluster_ctas == 1 || cluster_ctas == 2 ||
      cluster_ctas == 4 || cluster_ctas == 8)
    g_fps_force_cluster = cluster_ctas;
  return old;
}

int coda_furthest_point_sampling(int b, int n, int m, const float *xyz, int *idx,
                                 void *stream) {
  if (b < 0 || m < 0) return CODA_EINVAL;
  if (b == 0 || m == 0) return CODA_OK;  // sampling_gpu.cu:76: m <= 0 returns
  if (n <= 0 || !xyz || !idx) return CODA_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int bs_log2 = ref_block_size_log2(n);
  const int bs = 1 << bs_log2;
  const int R = (n + bs - 1) / bs;
  const long long P = (long long)R * bs;
  int cl = g_fps_force_cluster;
  if (cl == 0) cl = (P <= 4096) ? 1 : 8;
  int cl_log2 = 0;
  while ((1 << cl_log2) < cl) ++cl_log2;
  long long ppt = (P + ((long long)FPS_T << cl_log2) - 1) / ((long long)FPS_T << cl_log2);
  if (ppt > FPS_MAX_PPT && cl_log2 < 3) {  // widen before giving up on residency
    cl_log2 = 3;
    ppt = (P + (FPS_T << 3) - 1) / (FPS_T << 3);
  }
  if (ppt > FPS_MAX_PPT) {
    float *temp = nullptr;
    cudaError_t e = cudaMallocAsync(&temp, sizeof(float) * (size_t)b * n, s);
    if (e != cudaSuccess) return (int)e;
    fps_generic_kernel<<<b, 1024, 0, s>>>(n, m, bs_log2, R, xyz, temp, idx);
    const int st = launch_status();
    cudaFreeAsync(temp, s);
    return st;
  }
#define CODA_FPS_CASE(PPT_) \
  if (ppt <= PPT_) return launch_fps<PPT_>(b, n, m, bs_log2, R, cl_log2, xyz, idx, s);
  CODA_FPS_CASE(1)
  CODA_FPS_CASE(2)
  CODA_FPS_CASE(3)
  CODA_FPS_CASE(4)
  CODA_FPS_CASE(5)
  CODA_FPS_CASE(6)
  CODA_FPS_CASE(8)
  CODA_FPS_CASE(10)
  CODA_FPS_CASE(12)
  CODA_FPS_CASE(16)
#undef CODA_FPS_CASE
  return CODA_ETOOLARGE;
}

int coda_gather_points(int b, int c, int n, int m, const float *points,
                       const int *idx, float *out, void *stream) {
  if (b < 0 || c < 0 || m < 0 || n < 0) return CODA_EINVAL;
  if (b == 0 || c == 0 || m == 0) return CODA_OK;
  if (!points || !idx || !out || n == 0 || c > 65535 || b > 65535) return CODA_EINVAL;
  gather_points_kernel<<<dim3((m + 255) / 256, c, b), 256, 0, (cudaStream_t)stream>>>(
      c, n, m, points, idx, out);
  return launch_status();
}

int coda_gather_points_grad(int b, int c, int n, int m, const float *grad_out,
                            const int *idx, float *grad_points, void *stream) {
  if (b < 0 || c < 0 || m < 0 || n < 0) return CODA_EINVAL;
  if (b == 0 || c == 0 || m == 0) return CODA_OK;
  if (!grad_out || !idx || !grad_points || n == 0 || c > 65535 || b > 65535) return CODA_EINVAL;
  gather_points_grad_kernel<<<dim3((m + 255) / 256, c, b), 256, 0, (cudaStream_t)stream>>>(
      c, n, m, grad_out, idx, grad_points);
  return launch_status();
}

static int ball_query_impl(bool group, int b, int n, int m, float radius, int nsample,
                           int normalize, const float *xyz, const float *new_xyz,
                           int *idx, float *grouped, void *stream) {
  if (b < 0 || n < 0 || m < 0 || nsample < 0) return CODA_EINVAL;
  if (b == 0 || m == 0 || nsample == 0) return CODA_OK;
  if (!new_xyz || !idx || (n > 0 && !xyz) || (group && !grouped) || b > 65535) return CODA_EINVAL;
  if (group && n == 0) return CODA_EINVAL;  // index 0 would be gathered from an empty scene
  const size_t smem = BQ_TILE * 3 * sizeof(float) + (size_t)BQ_WARPS * nsample * sizeof(int);
  if (smem > 200 * 1024) return CODA_ETOOLARGE;
  const float radius2 = radius * radius;  // ball_query_gpu.cu:24, fp32
  const float inv_radius = 1.0f / radius;
  const dim3 grid((m + BQ_WARPS - 1) / BQ_WARPS, b);
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e;
  if (group) {
    e = cudaFuncSetAttribute(ball_query_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    ball_query_kernel<true><<<grid, BQ_T, smem, s>>>(n, m, radius2, nsample, normalize, inv_radius,
                                                    xyz, new_xyz, idx, grouped);
  } else {
    e = cudaFuncSetAttribute(ball_query_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    ball_query_kernel<false><<<grid, BQ_T, smem, s>>>(n, m, radius2, nsample, 0, 1.0f, xyz, new_xyz,
                                                     idx, nullptr);
  }
  return launch_status();
}

int coda_ball_query(int b, int n, int m, float radius, int nsample,
                    const float *new_xyz, const float *xyz, int *idx, void *stream) {
  return ball_query_impl(false, b, n, m, radius, nsample, 0, xyz, new_xyz, idx, nullptr, stream);
}

int coda_query_and_group_xyz(int b, int n, int m, float radius, int nsample,
                             int normalize, const float *xyz, const float *new_xyz,
                             int *idx, float *grouped, void *stream) {
  return ball_query_impl(true, b, n, m, radius, nsample, normalize, xyz, new_xyz, idx, grouped, stream);
}

int coda_group_points(int b, int c, int n, int npoints, int nsample,
                      const float *points, const int *idx, float *out, void *stream) {
  if (b < 0 || c < 0 || n < 0 || npoints < 0 || nsample < 0) return CODA_EINVAL;
  const long long ms = (long long)npoints * nsample;
  if (b == 0 || c == 0 || ms == 0) return CODA_OK;
  if (!points || !idx || !out || n == 0 || b > 65535 || ms > 0x7fffffffLL) return CODA_EINVAL;
  const int cpb = pick_c_per_block(c, ms, b);
  const dim3 grid((unsigned)((ms + 255) / 256), (c + cpb - 1) / cpb, b);
  group_points_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(c, n, (int)ms, cpb, points, idx, out);
  return launch_status();
}

int coda_group_points_grad(int b, int c, int n, int npoints, int nsample,
                           const float *grad_out, const int *idx, float *grad_points,
                           void *stream) {
  if (b < 0 || c < 0 || n < 0 || npoints < 0 || nsample < 0) return CODA_EINVAL;
  const long long ms = (long long)npoints * nsample;
  if (b == 0 || c == 0 || ms == 0) return CODA_OK;
  if (!grad_out || !idx || !grad_points || n == 0 || b > 65535 || ms > 0x7fffffffLL) return CODA_EINVAL;
  const int cpb = pick_c_per_block(c, ms, b);
  const dim3 grid((unsigned)((ms + 255) / 256), (c + cpb - 1) / cpb, b);
  group_points_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(c, n, (int)ms, cpb, grad_out, idx,
                                                                 grad_points);
  return launch_status();
}

int coda_three_nn(int b, int n, int m, const float *unknown, const float *known,
                  float *dist2, int *idx, void *stream) {
  if (b < 0 || n < 0 || m < 0) return CODA_EINVAL;
  if (b == 0 || n == 0) return CODA_OK;
  if (!unknown || !dist2 || !idx || (m > 0 && !known) || b > 65535) return CODA_EINVAL;
  three_nn_kernel<<<dim3((n + NN_T - 1) / NN_T, b), NN_T, 0, (cudaStream_t)stream>>>(
      n, m, unknown, known, dist2, idx);
  return launch_status();
}

int coda_three_interpolate(int b, int c, int m, int n, const float *points,
                           const int *idx, const float *weight, float *out, void *stream) {
  if (b < 0 || c < 0 || m < 0 || n < 0) return CODA_EINVAL;
  if (b == 0 || c == 0 || n == 0) return CODA_OK;
  if (!points || !idx || !weight || !out || m == 0 || b > 65535) return CODA_EINVAL;
  const int cpb = pick_c_per_block(c, n, b);
  const dim3 grid((n + 255) / 256, (c + cpb - 1) / cpb, b);
  three_interpolate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(c, m, n, cpb, points, idx, weight, out);
  return launch_status();
}

int coda_three_interpolate_grad(int b, int c, int n, int m, const float *grad_out,
                                const int *idx, const float *weight, float *grad_points,
                                void *stream) {
  if (b < 0 || c < 0 || m < 0 || n < 0) return CODA_EINVAL;
  if (b == 0 || c == 0 || n == 0) return CODA_OK;
  if (!grad_out || !idx || !weight || !grad_points || m == 0 || b > 65535) return CODA_EINVAL;
  const int cpb = pick_c_per_block(c, n, b);
  const dim3 grid((n + 255) / 256, (c + cpb - 1) / cpb, b);
  three_interpolate_grad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(c, n, m, cpb, grad_out, idx,
                                                                      weight, grad_points);
  return launch_status();
}

}  // extern "C"
