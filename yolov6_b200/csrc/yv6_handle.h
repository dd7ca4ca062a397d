// yv6_handle.h -- per-device context behind the opaque `yv6_handle` of include/yv6.h.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>

typedef CUresult (*yv6_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

struct yv6_handle {
  int device;
  int num_sms;
  int max_smem_optin;              // bytes of dynamic shared memory a CTA may opt in to
  yv6_encode_tiled_fn encode_tiled;  // resolved through cudaGetDriverEntryPoint (no -lcuda)
  void* scratch;                   // device scratch for kernels that need counters / partials
  size_t scratch_bytes;
  unsigned configured;             // YV6_CFG_* bits: cudaFuncSetAttribute is per device, so the flags live in the handle
  int max_clusters;                // co-resident 2-CTA clusters of the conv kernel (one CTA per SM); 0 = pairs unavailable
};

enum { YV6_CFG_CONV = 1u, YV6_CFG_WGRAD = 2u, YV6_CFG_NMS = 4u, YV6_CFG_BN = 8u, YV6_CFG_TRAIN2 = 16u, YV6_CFG_POOL = 32u, YV6_CFG_SELROWS = 64u, YV6_CFG_POOL16 = 128u, YV6_CFG_STEM = 256u, YV6_CFG_METRICS = 512u, YV6_CFG_COCO = 1024u, YV6_CFG_POOLF16 = 2048u };

// Every entry point runs on the handle's device whatever the caller's current device is, and leaves the
// caller's current device untouched (several handles / GPUs in one process, nn.DataParallel-style callers).
struct yv6_device_guard {
  int prev = -1;
  bool switched = false;
  explicit yv6_device_guard(const yv6_handle* h) {
    if (h != nullptr && cudaGetDevice(&prev) == cudaSuccess && prev != h->device) switched = (cudaSetDevice(h->device) == cudaSuccess);
  }
  ~yv6_device_guard() {
    if (switched) cudaSetDevice(prev);
  }
  yv6_device_guard(const yv6_device_guard&) = delete;
  yv6_device_guard& operator=(const yv6_device_guard&) = delete;
};
