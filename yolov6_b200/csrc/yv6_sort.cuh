// yv6_sort.cuh -- stable LSD radix sort of (uint64 key, uint32 value) pairs and CTA-wide scans, shared by the PR metric
// (yv6_metrics.cu) and the COCO box evaluation (yv6_cocoeval.cu).
//
// rs_pass sorts by one 8-bit digit of the key (bits shift .. shift + 7), stably; LSD passes from the lowest digit up give a
// stable sort by the digits passed.  The kernels live in an unnamed namespace: each including file gets its own copy.
#pragma once
#include <cstdint>

#include <cuda_runtime.h>

namespace yv6 {
namespace {

constexpr int kRsThreads = 256, kRsItems = 16, kRsTile = kRsThreads * kRsItems, kRsWarps = kRsThreads / 32;

__global__ void __launch_bounds__(kRsThreads) rs_hist_kernel(const uint64_t* __restrict__ keys, int64_t N, int shift, int nblk,
                                                             uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kRsTile;
  for (int i = threadIdx.x; i < kRsTile; i += kRsThreads)
    if (base + i < N) atomicAdd(&h[(keys[base + i] >> shift) & 255], 1u);
  __syncthreads();
  hist[(int64_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

// exclusive scan of n counters in one CTA (n = 256 * blocks of the sort, a few hundred thousand at most)
__global__ void __launch_bounds__(1024) rs_scan_kernel(uint32_t* __restrict__ v, int64_t n) {
  __shared__ uint32_t s_w[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t per = (n + 1023) / 1024, lo = min(n, (int64_t)tid * per), hi = min(n, lo + per);
  uint32_t sum = 0;
  for (int64_t i = lo; i < hi; ++i) sum += v[i];
  uint32_t x = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = s_w[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    s_w[lane] = w;
  }
  __syncthreads();
  uint32_t run = x - sum + (warp > 0 ? s_w[warp - 1] : 0);
  for (int64_t i = lo; i < hi; ++i) {
    const uint32_t c = v[i];
    v[i] = run;
    run += c;
  }
}

// stable scatter: rounds of 256 consecutive keys; within a warp __match_any gives the rank among equal digits, warps are
// ordered through per-warp digit counts
__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                                uint64_t* __restrict__ kout, uint32_t* __restrict__ vout, int64_t N,
                                                                int shift, int nblk, const uint32_t* __restrict__ hist) {
  __shared__ uint32_t s_cnt[kRsWarps][256];
  __shared__ uint32_t s_run[256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  s_run[tid] = hist[(int64_t)tid * nblk + blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * kRsTile;
  for (int r = 0; r < kRsItems; ++r) {
#pragma unroll
    for (int w = 0; w < kRsWarps; ++w) s_cnt[w][tid] = 0;
    __syncthreads();
    const int64_t i = base + (int64_t)r * kRsThreads + tid;
    const bool valid = i < N;
    const uint64_t k = valid ? kin[i] : 0;
    const uint32_t d = valid ? (uint32_t)(k >> shift) & 255u : 256u;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) s_cnt[warp][d] = __popc(peers);
    __syncthreads();
    uint32_t run = s_run[tid];
#pragma unroll
    for (int w = 0; w < kRsWarps; ++w) {
      const uint32_t c = s_cnt[w][tid];
      s_cnt[w][tid] = run;
      run += c;
    }
    s_run[tid] = run;
    __syncthreads();
    if (valid) {
      const uint32_t pos = s_cnt[warp][d] + rank;
      kout[pos] = k;
      vout[pos] = vin[i];
    }
    __syncthreads();
  }
}

// counters the histogram of one pass over N keys needs
inline int64_t rs_hist_words(int64_t N) { return (int64_t)256 * ((N + kRsTile - 1) / kRsTile); }

// one stable pass by the digit at `shift`: (kin, vin) -> (kout, vout); hist holds rs_hist_words(N) counters
inline void rs_pass(const uint64_t* kin, const uint32_t* vin, uint64_t* kout, uint32_t* vout, int64_t N, int shift, uint32_t* hist,
                    cudaStream_t s) {
  const int nblk = (int)((N + kRsTile - 1) / kRsTile);
  rs_hist_kernel<<<nblk, kRsThreads, 0, s>>>(kin, N, shift, nblk, hist);
  rs_scan_kernel<<<1, 1024, 0, s>>>(hist, (int64_t)256 * nblk);
  rs_scatter_kernel<<<nblk, kRsThreads, 0, s>>>(kin, vin, kout, vout, N, shift, nblk, hist);
}

// exclusive prefix sum over the CTA; returns the CTA total in *total
__device__ __forceinline__ int block_excl_sum(int v, int* s_w, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  int off = 0, tot = 0;
  for (int w = 0; w < nw; ++w) {
    off += w < warp ? s_w[w] : 0;
    tot += s_w[w];
  }
  *total = tot;
  return off + x - v;
}

// max over the threads with a higher index (exclusive suffix max); every value is >= 0, the empty max is 0
__device__ __forceinline__ double block_excl_sufmax(double v, double* s_w, double* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  double x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const double y = __shfl_down_sync(0xffffffffu, x, o);
    if (lane + o < 32) x = fmax(x, y);
  }
  double nxt = __shfl_down_sync(0xffffffffu, x, 1);
  if (lane == 31) nxt = 0.0;
  __syncthreads();
  if (lane == 0) s_w[warp] = x;
  __syncthreads();
  double later = 0.0, tot = 0.0;
  for (int w = 0; w < nw; ++w) {
    if (w > warp) later = fmax(later, s_w[w]);
    tot = fmax(tot, s_w[w]);
  }
  *total = tot;
  return fmax(nxt, later);
}

}  // namespace
}  // namespace yv6
