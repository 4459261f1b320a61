// Shared device/host helpers for the coda_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define CODA_OK 0
#define CODA_EINVAL (-1)
#define CODA_ETOOLARGE (-2)

namespace coda {

__host__ inline int launch_status() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? CODA_OK : (int)e;
}

// Raise kernel Kern's dynamic shared-memory limit to `bytes` on the first call; later calls do nothing, so `bytes` must
// cover every launch of Kern.  The flag is one per kernel (Kern is the function pointer: the instances of a kernel
// template share one function type).
template <auto Kern>
__host__ inline int raise_smem_limit(int bytes) {
  static bool done = false;
  if (!done) {
    const cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return (int)e;
    done = true;
  }
  return CODA_OK;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// ---- mbarrier (shared::cta) -------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(count)
               : "memory");
}
__device__ __forceinline__ void mbar_fence_init_cluster() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar,
                                                      uint32_t bytes) {
  asm volatile(
      "mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
          smem_u32(bar)),
      "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// Wait for warps that are MANY and not on the critical path alone (GEMM transform / epilogue warps): a
// three-instruction loop around try_wait with a suspend-time hint, so that a waiting warp sleeps in hardware instead
// of spinning through select / compare / address-conversion instructions.  ncu on the weight-gradient GEMM: the spin
// loops of the sixteen transform warps were a fifth of all issued instructions and took issue slots from the warps
// that had work.  Single-warp roles (TMA producer, MMA issuer) keep the plain spin: lowest wake-up latency.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t *bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra DONE%=;\n\t"
      "bra LAB_WAIT%=;\n\t"
      "DONE%=:\n\t"
      "}"
      :
      : "r"(addr), "r"(parity), "r"(0x989680u)
      : "memory");
}

// Map a local shared-memory address to the same offset in CTA `rank` of the
// cluster (shared::cluster window).
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;"
               : "=r"(r)
               : "r"(local_addr), "r"(rank));
  return r;
}

// 16-byte asynchronous store into a peer CTA's shared memory that completes
// `16` transaction bytes on that CTA's mbarrier.
__device__ __forceinline__ void st_async_v4(uint32_t remote_addr,
                                            uint32_t remote_mbar, uint32_t a,
                                            uint32_t b, uint32_t c,
                                            uint32_t d) {
  asm volatile(
      "st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 "
      "[%0], {%2, %3, %4, %5}, [%1];" ::"r"(remote_addr),
      "r"(remote_mbar), "r"(a), "r"(b), "r"(c), "r"(d)
      : "memory");
}

}  // namespace coda
