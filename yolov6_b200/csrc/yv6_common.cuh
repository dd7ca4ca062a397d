// yv6_common.cuh -- shared helpers for the yolov6_b200 sm_90a kernels.
//
// Error plumbing for the C-ABI (include/yv6.h) plus thin inline-PTX wrappers for
// the Hopper primitives the kernels use: mbarrier and TMA (cp.async.bulk.tensor).
// The wgmma wrappers live in yv6_wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/yv6.h"

// ----------------------------------------------------------------------------------------------
// error plumbing
// ----------------------------------------------------------------------------------------------
void yv6_set_error(const char* fmt, ...);

#define YV6_CHECK_CUDA(expr)                                                          \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      yv6_set_error("%s:%d CUDA error %d (%s) in `%s`", __FILE__, __LINE__, (int)_e,  \
                    cudaGetErrorString(_e), #expr);                                   \
      (void)cudaGetLastError(); /* a non-sticky error must not be blamed on the next call */ \
      return YV6_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

#define YV6_REQUIRE(cond, ...)                                                        \
  do {                                                                                \
    if (!(cond)) {                                                                    \
      yv6_set_error(__VA_ARGS__);                                                     \
      return YV6_ERR_ARG;                                                             \
    }                                                                                 \
  } while (0)

// ----------------------------------------------------------------------------------------------
// device-side PTX wrappers
// ----------------------------------------------------------------------------------------------
namespace yv6 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// One lane of a fully converged warp (always the same lane for the full mask).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin with a watchdog: a mis-programmed pipeline must trap (-> cudaErrorLaunchFailure on the
// host, surfaced as RuntimeError) instead of hanging the GPU.
//
// Rule: no function call may appear in a kernel that issues wgmma -- no __noinline__ helper, no printf, no assert.
// ptxas cannot keep an asynchronous wgmma pipeline across a call, so it serializes EVERY wgmma of the kernel (warning
// C7510: each MMA waits for the previous one to complete).  The watchdog is therefore fully inline and ends in __trap();
// the diagnostic line is opt-in (-DYV6_WATCHDOG_PRINTF) for debugging builds only, as it brings the serialization back.  tests/test_sass_wgmma.py checks
// the built library for calls and serialized MMAs.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3fff) == 0) {
      uint64_t now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) {  // 4 s
#ifdef YV6_WATCHDOG_PRINTF
        if ((threadIdx.x & 31) == 0) printf("yv6: mbarrier wait timeout block %d warp %d\n", blockIdx.x, threadIdx.x >> 5);
#endif
        __trap();
      }
    }
  }
}

// ---- thread block clusters ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at this shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile(
      "{\n"
      ".reg .b32 remote;\n"
      "mapa.shared::cluster.u32 remote, %0, %1;\n"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [remote];\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(rank)
      : "memory");
}

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "r"(c4)
      : "memory");
}

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case YV6_ACT_RELU: return fmaxf(v, 0.f);
    case YV6_ACT_SILU: return v / (1.f + expf(-v));
    case YV6_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case YV6_ACT_HARDSWISH: return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
    case YV6_ACT_HARDSIGMOID: return fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
    default: return v;
  }
}

}  // namespace yv6
