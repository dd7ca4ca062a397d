// yv6_conv_wgrad.cu -- weight gradient of a 1x1 / 3x3 convolution on Hopper warpgroup tensor cores (wgmma, sm_90a).
//
//   dW[co][r][s][ci] = sum over output pixels (n,ho,wo) of dY[n,ho,wo,co] * X[n, ho*st + r - pad, wo*st + s - pad, ci]
//
// i.e. what autograd computes for `F.conv2d` in the reference's training step (Trainer.train_in_steps,
// yolov6/core/engine.py:142-176 -> cuDNN wgrad).  GEMM view per filter tap: M = Cout, N = Cin, K = pixels.
// Both operands are read straight from the NHWC activations by TMA as [pixels][channels] boxes; that
// shared-memory image is the canonical *MN-major* swizzled wgmma layout (channels contiguous, 8 pixel rows
// per swizzle atom), so no transpose is ever materialised:
//   A = dY box  (K = pixels x M = 64-wide Cout blocks),
//   B = X box shifted by the tap (zero fill = padding, elementStrides = conv stride).
// One CTA owns a (Cout tile of 128, Cin tile, tap group, pixel range) unit: consumer warpgroup w accumulates Cout rows
// 64 w .. 64 w + 63 x NT columns per tap in registers over its pixel tiles and adds the result to dW with fp32 reductions
// (split-K over the pixel ranges).  Warp 0 = TMA producer, warpgroups 1-2 = wgmma consumers.
#include <algorithm>
#include <cstdlib>

#include "yv6_common.cuh"
#include "yv6_handle.h"
#include "yv6_wgmma.cuh"

namespace yv6 {

constexpr int kWgThreads = 384;
constexpr int kWgMaxStages = 8;
constexpr int kWgFixedSmem = 1024 /* alignment */ + 512 /* barriers */;

struct WgParams {
  int32_t BW, BH, PT;                 // pixel box, BW*BH == PT (128 or 64): the K extent of one pipeline stage
  int32_t tiles_w, tiles_h, tiles_i, ptiles;
  int32_t co_tiles, ci_tiles, taps, kw, ksplit;
  int32_t T, tap_groups;              // taps per unit (1, or 3 = one filter row) and taps / T
  int32_t Cout, Cin, stride, pad;
  int32_t a_loaded;                   // 64-wide dY blocks TMA fetches = consumer warpgroups at work (1 if Cout <= 64)
  int32_t b_blocks, b_blk_elems, b_blk_bytes;  // X blocks of 64/32/16 channels
  int32_t NT;                         // wgmma N = b_blocks * b_blk_elems
  int32_t stages, a_stage_bytes, b_tap_bytes, b_stage_bytes;
  float* dw;                          // fp32 [Cout][kh*kw][Cin]
};

__device__ __forceinline__ void wg_tma_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// NT = wgmma N (Cin tile), T = taps per unit, PT = pixels per stage (K extent)
template <int NT, int T>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgParams p) {
  constexpr int PT = (T == 3) ? 64 : 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + (size_t)p.stages * p.a_stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + (size_t)p.stages * p.b_stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kWgMaxStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // unit decode: tap group fastest, then channel tiles, then the pixel range -- CTAs that run at the same time read the SAME
  // pixels of dY / X for different taps / channel tiles, so each operand byte is fetched from DRAM once and then served by L2
  int u = blockIdx.x;
  const int tg = u % p.tap_groups; u /= p.tap_groups;
  const int ci_t = u % p.ci_tiles; u /= p.ci_tiles;
  const int co_t = u % p.co_tiles; u /= p.co_tiles;
  const int ks = u;
  const int tap0 = tg * T;
  const int per = (p.ptiles + p.ksplit - 1) / p.ksplit;
  const int pt0 = ks * per, pt1 = min(p.ptiles, pt0 + per);
  const int npt = max(0, pt1 - pt0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], (uint32_t)p.a_loaded); }
    fence_mbar_init();
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
  }
  __syncthreads();
  const uint32_t a_blk_bytes = (uint32_t)PT * 128u;                  // one 64-channel dY block: PT pixel rows of 128 bytes

  if (warp == 0) {
    const uint32_t tx = (uint32_t)p.a_loaded * a_blk_bytes + (uint32_t)(T * p.b_blocks * PT * p.b_blk_bytes);
    int stage = 0;
    uint32_t phase = 0;
    for (int pt = pt0; pt < pt1; ++pt) {
      int m = pt;
      const int tw = m % p.tiles_w; m /= p.tiles_w;
      const int th = m % p.tiles_h;
      const int ti = m / p.tiles_h;
      const int w0 = tw * p.BW, h0 = th * p.BH;
      mbar_wait(&empty[stage], phase ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&full[stage], tx);
        for (int j = 0; j < p.a_loaded; ++j)
          wg_tma_4d(sA + (size_t)stage * p.a_stage_bytes + (size_t)j * a_blk_bytes, &tmDY, &full[stage], co_t * 128 + j * 64, w0, h0, ti);
        for (int t = 0; t < T; ++t) {
          const int tap = tap0 + t;
          const int r = tap / p.kw, sx = tap - r * p.kw;
          uint8_t* dst = sB + (size_t)stage * p.b_stage_bytes + (size_t)t * p.b_tap_bytes;
          for (int j = 0; j < p.b_blocks; ++j)
            wg_tma_4d(dst + (size_t)j * PT * p.b_blk_bytes, &tmX, &full[stage], ci_t * NT + j * p.b_blk_elems,
                      w0 * p.stride + sx - p.pad, h0 * p.stride + r - p.pad, ti);
        }
      }
      __syncwarp();
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
  } else if (warp >= 4 && (warp >> 2) - 1 < p.a_loaded) {
    // consumer warpgroup wg: Cout rows co_t * 128 + 64 wg + (0 .. 63).  Both operands MN-major (wgmma transpose bits set):
    // LBO = bytes between channel blocks, SBO = bytes between 8-pixel-row groups; a K step of 16 pixels = two such groups.
    const int wg = (warp >> 2) - 1;
    float acc[T][NT / 2];
    const uint64_t da = wgmma_desc(a_blk_bytes, 1024u, 1u);
    const uint64_t db = wgmma_desc((uint32_t)(PT * p.b_blk_bytes), (uint32_t)(8 * p.b_blk_bytes), wgmma_layout(p.b_blk_bytes));
    const uint32_t a_base = (smem_u32(sA) + (uint32_t)wg * a_blk_bytes) >> 4, b_base = smem_u32(sB) >> 4;
    const uint32_t a_step = (uint32_t)p.a_stage_bytes >> 4, b_step = (uint32_t)p.b_stage_bytes >> 4, b_tap = (uint32_t)p.b_tap_bytes >> 4;
    const uint32_t a_k = 2048u >> 4, b_k = (uint32_t)(16 * p.b_blk_bytes) >> 4;
    const bool arrive_lane = ((warp & 3) == 0) && lane == 0;
#pragma unroll
    for (int t = 0; t < T; ++t)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[t][i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int it = 0; it < npt; ++it) {
      mbar_wait(&full[stage], phase);
      const uint64_t ad = da | (uint64_t)(a_base + (uint32_t)stage * a_step);
      const uint64_t bd = db | (uint64_t)(b_base + (uint32_t)stage * b_step);
      wgmma_fence();
#pragma unroll
      for (int t = 0; t < T; ++t) {
#pragma unroll
        for (int k = 0; k < PT / 16; ++k)
          Wgmma<NT, 1, 1>::mma(acc[t], ad + (uint64_t)(k * a_k), bd + (uint64_t)(t * b_tap + k * b_k), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && arrive_lane) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < T; ++t) wgmma_fence_operand(acc[t]);
    if (npt > 0) {
      // fragment: acc[t][4 j + 2 i + c] = dW row (co) 16 (warp % 4) + lane / 4 + 8 i, column (ci) 8 j + 2 (lane % 4) + c
      const int co0 = co_t * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int ci0 = ci_t * NT + 2 * (lane & 3);
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const int tap = tap0 + t;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int co = co0 + 8 * i;
          if (co >= p.Cout) continue;
          float* row = p.dw + ((int64_t)co * p.taps + tap) * p.Cin;
#pragma unroll
          for (int j = 0; j < NT / 8; ++j) {
            const int ci = ci0 + 8 * j;
            if (ci < p.Cin) {          // Cin % 16 == 0 and ci is even: ci + 1 < Cin as well
              atomicAdd(row + ci, acc[t][4 * j + 2 * i]);
              atomicAdd(row + ci + 1, acc[t][4 * j + 2 * i + 1]);
            }
          }
        }
      }
    }
  }
}

}  // namespace yv6

using namespace yv6;

using WgradKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const WgParams);
// [NT index: 16, 32, 64, 128][T == 3]
static const WgradKernelFn kWgradKernels[4][2] = {{conv_wgrad_kernel<16, 1>, conv_wgrad_kernel<16, 3>},
                                                  {conv_wgrad_kernel<32, 1>, conv_wgrad_kernel<32, 3>},
                                                  {conv_wgrad_kernel<64, 1>, conv_wgrad_kernel<64, 3>},
                                                  {conv_wgrad_kernel<128, 1>, nullptr}};

// The launch plan of one weight gradient on a device with `num_sms` SMs and `max_smem_optin` bytes of opt-in shared memory:
// tile shapes, pipeline depth and the split-K over pixel ranges.  Shared by yv6_conv_wgrad and yv6_wgrad_plan_host.
static int plan_wgrad(int num_sms, int max_smem_optin, const yv6_wgrad_desc* d, WgParams& p) {
  YV6_REQUIRE(d->Cin > 0 && d->Cin % 16 == 0 && d->x_c_total % 8 == 0 && d->dy_c_total % 8 == 0, "wgrad: channel counts");
  YV6_REQUIRE(d->kh == d->kw && (d->kh == 1 || d->kh == 3), "wgrad: kernel %dx%d unsupported", d->kh, d->kw);
  YV6_REQUIRE(d->stride == 1 || d->stride == 2, "wgrad: stride %d", d->stride);
  const int Ho = (d->H + 2 * d->pad - d->kh) / d->stride + 1, Wo = (d->W + 2 * d->pad - d->kw) / d->stride + 1;
  memset(&p, 0, sizeof(p));
  p.Cout = d->Cout; p.Cin = d->Cin; p.stride = d->stride; p.pad = d->pad;
  p.taps = d->kh * d->kw; p.kw = d->kw;
  p.dw = d->dw;
  // 3x3: one CTA accumulates the three taps of a filter row -- they share the dY tile, which cuts the L2 -> SM operand
  // stream per MMA by 1.5x (128 channels) to 2.3x (64 channels); the Cin tile is then at most 64 wide (3 x 32 accumulator
  // registers per thread), otherwise at most 128.
  p.T = (p.taps == 9 && d->force_taps != 1) ? 3 : 1;
  const int nt_max = (p.T == 3) ? 64 : 128;
  p.NT = 16;
  while (p.NT < nt_max && p.NT < d->Cin) p.NT <<= 1;          // channels past Cin are zero filled by TMA and never stored
  p.ci_tiles = (d->Cin + p.NT - 1) / p.NT;
  p.b_blk_elems = std::min(64, p.NT);
  p.b_blk_bytes = p.b_blk_elems * 2;
  p.b_blocks = p.NT / p.b_blk_elems;
  p.tap_groups = p.taps / p.T;
  p.PT = (p.T == 3) ? 64 : 128;
  // pixel box: exactly PT rows (partial boxes are zero filled by TMA, so the K sum stays exact)
  long best = -1;
  for (int bw = 1; bw <= p.PT; bw <<= 1) {
    const int bh = p.PT / bw;
    if (bw * d->stride > 256 || bh * d->stride > 256) continue;
    const long t = (long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * d->N;
    if (best < 0 || t < best || (t == best && bw > p.BW)) { best = t; p.BW = bw; p.BH = bh; }
  }
  p.tiles_w = (Wo + p.BW - 1) / p.BW; p.tiles_h = (Ho + p.BH - 1) / p.BH; p.tiles_i = d->N;
  p.ptiles = p.tiles_w * p.tiles_h * p.tiles_i;
  p.a_loaded = (d->Cout <= 64) ? 1 : 2;     // the second consumer warpgroup (Cout rows 64..127 of the tile) idles for Cout <= 64
  p.co_tiles = (d->Cout + 127) / 128;
  p.a_stage_bytes = p.a_loaded * p.PT * 128;
  p.b_tap_bytes = ((p.b_blocks * p.PT * p.b_blk_bytes + 1023) / 1024) * 1024;
  p.b_stage_bytes = p.T * p.b_tap_bytes;
  const int budget = max_smem_optin - kWgFixedSmem;
  p.stages = std::min(kWgMaxStages, budget / (p.a_stage_bytes + p.b_stage_bytes));
  YV6_REQUIRE(p.stages >= 2, "wgrad: not enough shared memory");
  const int base_units = p.co_tiles * p.ci_tiles * p.tap_groups;
  // split-K over pixel ranges: the kernel is bound by the L2 -> shared-memory operand stream of each CTA (measured: the time
  // per 64-pixel stage does not depend on how many CTAs run), so it wants exactly two full waves of CTAs -- one unit more than
  // a multiple of the SM count costs a whole extra wave -- with at least ~8 stages of work each (every extra split adds a
  // pass of fp32 reductions over the weight tensor)
  const int min_tiles = 8 * 128 / p.PT;
  p.ksplit = std::max(1, std::min((p.ptiles + min_tiles - 1) / min_tiles, std::max(1, 2 * num_sms / base_units)));
  if (d->force_ksplit > 0) p.ksplit = std::min(p.ptiles, d->force_ksplit);
  return YV6_OK;
}

extern "C" int yv6_wgrad_plan_host(int num_sms, int max_smem_optin, const yv6_wgrad_desc* d, int32_t* out10) {
  YV6_REQUIRE(d != nullptr && out10 != nullptr, "wgrad_plan_host: null argument");
  YV6_REQUIRE(num_sms > 0 && max_smem_optin > 0, "wgrad_plan_host: bad device properties");
  WgParams p;
  const int rc = plan_wgrad(num_sms, max_smem_optin, d, p);
  if (rc != YV6_OK) return rc;
  const int per = (p.ptiles + p.ksplit - 1) / p.ksplit;
  out10[0] = p.NT;
  out10[1] = p.T;
  out10[2] = p.PT;
  out10[3] = p.BW;
  out10[4] = p.BH;
  out10[5] = p.ptiles;
  out10[6] = p.ksplit;
  out10[7] = per * p.PT;
  out10[8] = p.co_tiles * p.ci_tiles * p.tap_groups * p.ksplit;
  out10[9] = p.stages * (p.a_stage_bytes + p.b_stage_bytes) + kWgFixedSmem;
  return YV6_OK;
}

extern "C" int yv6_conv_wgrad(yv6_handle* h, const yv6_wgrad_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->x && d->dy && d->dw, "wgrad: null argument");
  YV6_REQUIRE(h->encode_tiled != nullptr, "wgrad: cuTensorMapEncodeTiled unavailable");
  WgParams p;
  { const int rc = plan_wgrad(h->num_sms, h->max_smem_optin, d, p); if (rc != YV6_OK) return rc; }
  const int Ho = (d->H + 2 * d->pad - d->kh) / d->stride + 1, Wo = (d->W + 2 * d->pad - d->kw) / d->stride + 1;
  const int units = p.co_tiles * p.ci_tiles * p.tap_groups * p.ksplit;

  CUtensorMap tmDY, tmX;
  {
    cuuint64_t dims[4] = {(cuuint64_t)d->Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)d->N};
    const uint64_t pix = (uint64_t)d->dy_c_total * 2;
    cuuint64_t strides[3] = {pix, pix * Wo, pix * Wo * Ho};
    cuuint32_t box[4] = {64, (cuuint32_t)p.BW, (cuuint32_t)p.BH, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult cr = h->encode_tiled(&tmDY, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->dy), dims, strides, box, es,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { yv6_set_error("wgrad: cuTensorMapEncodeTiled(dY) failed with %d", (int)cr); return YV6_ERR_CUDA; }
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
    const uint64_t pix = (uint64_t)d->x_c_total * 2;
    cuuint64_t strides[3] = {pix, pix * d->W, pix * d->W * d->H};
    cuuint32_t box[4] = {(cuuint32_t)p.b_blk_elems, (cuuint32_t)(p.BW * d->stride), (cuuint32_t)(p.BH * d->stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
    const CUtensorMapSwizzle sw = (p.b_blk_bytes == 128) ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : (p.b_blk_bytes == 64) ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult cr = h->encode_tiled(&tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->x), dims, strides, box, es,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { yv6_set_error("wgrad: cuTensorMapEncodeTiled(X) failed with %d", (int)cr); return YV6_ERR_CUDA; }
  }
  if (!(h->configured & YV6_CFG_WGRAD)) {
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 2; ++j)
        if (kWgradKernels[i][j] != nullptr)
          YV6_CHECK_CUDA(cudaFuncSetAttribute(kWgradKernels[i][j], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->max_smem_optin));
    h->configured |= YV6_CFG_WGRAD;
  }
  const size_t smem = (size_t)p.stages * (p.a_stage_bytes + p.b_stage_bytes) + kWgFixedSmem;
  const int nt_idx = p.NT == 16 ? 0 : p.NT == 32 ? 1 : p.NT == 64 ? 2 : 3;
  kWgradKernels[nt_idx][p.T == 3 ? 1 : 0]<<<units, kWgThreads, smem, (cudaStream_t)stream>>>(tmDY, tmX, p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
