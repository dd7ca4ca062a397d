// yv6_aux.cu -- the HBM-bound helpers around the conv kernel (sm_90a, CUDA cores):
//   * yv6_stem_fwd   : first 3x3 s2 conv on the 3-channel NCHW image (fp32 or uint8/255) -> NHWC bf16 (yv6_stem_fwd_f16: fp16)
//   * yv6_sppf_pool  : the three chained 5x5 max-pools of (CSP)SPPF written straight into concat slices
//   * yv6_head_decode: DFL expectation + ltrb -> xywh + x stride + [xywh, 1, cls] assembly
#include <type_traits>

#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace yv6 {

// ------------------------------------------------------------------------------------------------
// stem: reference RepVGGBlock / ConvBNSiLU `backbone.stem` (efficientrep.py:28-33) in deploy form,
// fused with the input conversion of Trainer.prepro_data / Inferer.process_image
// (engine.py:407-410, inferer.py:162-171: uint8 -> float / 255, NCHW).
// One thread = one output pixel, all Cout channels; the 27*Cout weights ride in the kernel
// parameter (constant bank) so every FFMA takes its weight operand straight from c[0][..].
// ------------------------------------------------------------------------------------------------
constexpr int kStemMaxCout = 64;
struct StemParams {
  const float* w;      // device fp32 [tap(r,s)][cin][cout] (27 x Cout)
  const float* b;      // device fp32 [Cout] or null
  const void* x;
  __nv_bfloat16* y;
  int64_t y_plane_stride;
  int32_t N, H, W, Ho, Wo;
  int32_t x_u8, act, planes;
  float in_scale;
};

// One thread = one output pixel x all COUT channels; the 27 x COUT weights sit in shared memory and are
// read as float4 broadcasts (every lane reads the same address).  Outputs are staged so that the global
// stores are full 16-byte vectors of consecutive pixels.
template <int COUT>
__global__ void __launch_bounds__(256) stem_kernel(const StemParams p) {
  __shared__ __align__(16) float sw[27 * COUT];
  __shared__ __align__(16) __nv_bfloat16 tile[256 * COUT];
  for (int i = threadIdx.x; i < 27 * COUT; i += 256) sw[i] = p.w[i];
  __syncthreads();
  const int64_t total = (int64_t)p.N * p.Ho * p.Wo;
  const int64_t pix0 = (int64_t)blockIdx.x * 256;
  const int64_t pix = pix0 + threadIdx.x;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = p.b ? p.b[c] : 0.f;
  if (pix < total) {
    const int wo = (int)(pix % p.Wo);
    const int ho = (int)((pix / p.Wo) % p.Ho);
    const int n = (int)(pix / ((int64_t)p.Wo * p.Ho));
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = 2 * ho - 1 + r;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int wi = 2 * wo - 1 + s;
        const bool ok = (hi >= 0) && (hi < p.H) && (wi >= 0) && (wi < p.W);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float v = 0.f;
          if (ok) {
            const int64_t idx = (((int64_t)n * 3 + c) * p.H + hi) * p.W + wi;
            v = p.x_u8 ? (float)__ldg(reinterpret_cast<const uint8_t*>(p.x) + idx) * p.in_scale
                       : __ldg(reinterpret_cast<const float*>(p.x) + idx);
          }
          const float4* wk = reinterpret_cast<const float4*>(&sw[((r * 3 + s) * 3 + c) * COUT]);
#pragma unroll
          for (int c4 = 0; c4 < COUT / 4; ++c4) {
            const float4 w4 = wk[c4];
            acc[4 * c4 + 0] = fmaf(v, w4.x, acc[4 * c4 + 0]);
            acc[4 * c4 + 1] = fmaf(v, w4.y, acc[4 * c4 + 1]);
            acc[4 * c4 + 2] = fmaf(v, w4.z, acc[4 * c4 + 2]);
            acc[4 * c4 + 3] = fmaf(v, w4.w, acc[4 * c4 + 3]);
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = act_apply(acc[c], p.act);
  }
  const int nvec = 256 * COUT / 8;
  const int64_t left = total - pix0;
  const int64_t valid_elems = (left < 256 ? left : (int64_t)256) * COUT;
  for (int pl = 0; pl < p.planes; ++pl) {
    if (pl) __syncthreads();
#pragma unroll
    for (int c = 0; c < COUT; c += 2) {
      __nv_bfloat162 v = __floats2bfloat162_rn(acc[c], acc[c + 1]);
      *reinterpret_cast<__nv_bfloat162*>(&tile[threadIdx.x * COUT + c]) = v;
      if (pl + 1 < p.planes) {
        acc[c] -= __low2float(v);
        acc[c + 1] -= __high2float(v);
      }
    }
    __syncthreads();
    uint4* dst = reinterpret_cast<uint4*>(p.y + pl * p.y_plane_stride + pix0 * COUT);
    const uint4* src = reinterpret_cast<const uint4*>(tile);
    for (int i = threadIdx.x; i < nvec; i += 256)
      if ((int64_t)i * 8 < valid_elems) dst[i] = src[i];
  }
}

// The 16-bit activation dtype T of the tensor-core stems (__nv_bfloat16, or __half in the fp16 mode): a pair of values rounded to
// it, and one m16n8k16 mma.sync on T operands with fp32 accumulation.
template <typename T>
__device__ __forceinline__ uint32_t stem_pack2(float a, float b) {
  if constexpr (std::is_same_v<T, __half>) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}
template <typename T>
__device__ __forceinline__ void stem_mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same_v<T, __half>)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Tensor-core stem for bf16 activations: the 3x3 stride-2 conv over 3 input channels is a GEMM with K = 27
// (padded to 32).  Persistent CTAs walk tiles of 8 output rows x 32 output columns; the 17 x 65 x 3 input
// patch is staged in shared memory as bf16 with 16-byte global loads, each warp owns one output row (two
// 16-pixel m-tiles) and gathers its mma.sync A fragments straight from the patch; the weights live in
// registers as B fragments for the whole kernel.  The work is bound by HBM (read the image once, write
// N*Ho*Wo*Cout bf16 once), so legacy mma.sync is ample; what matters is the instruction count per pixel.  T: the activation
// dtype (the body of stem_mma_kernel and stem_mma_f16_kernel below).
template <int COUT, typename T>
__device__ __forceinline__ void stem_mma_body(const StemParams& p) {
  constexpr int TH = 8, TW = 32, PH = 2 * TH + 1, PW = 2 * TW + 1, NT = COUT / 8;
  constexpr int PWP = 68;                                  // patch row pitch; element j of a row = input column wi0 + j - 1
  static_assert(PW + 1 <= PWP, "patch pitch");
  constexpr int PITCH = COUT * 2 + 16;                     // staged output row pitch (bytes): conflict-free
  __shared__ __align__(16) T patch[3 * PH * PWP];
  __shared__ __align__(16) uint8_t stage[8 * 32 * PITCH];
  const int tiles_w = (p.Wo + TW - 1) / TW, tiles_h = (p.Ho + TH - 1) / TH;
  const int num_tiles = tiles_w * tiles_h * p.N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;

  // ---- weights -> B fragments (bf16), bias -> registers; once per CTA ----
  uint32_t bfrag[NT][2][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int k = ks * 16 + h2 * 8 + 2 * t, nn = nt * 8 + g;
        const float w0 = (k < 27) ? __ldg(p.w + k * COUT + nn) : 0.f;
        const float w1 = (k + 1 < 27) ? __ldg(p.w + (k + 1) * COUT + nn) : 0.f;
        bfrag[nt][ks][h2] = stem_pack2<T>(w0, w1);
      }
  float bias[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bias[nt][0] = p.b ? __ldg(p.b + nt * 8 + 2 * t) : 0.f;
    bias[nt][1] = p.b ? __ldg(p.b + nt * 8 + 2 * t + 1) : 0.f;
  }
  // ---- A-fragment gather offsets of this thread: k -> (channel, tap row, tap column) ----
  int koff[2][2][2];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = ks * 16 + h2 * 8 + 2 * t + e;
        const int tap = k / 3, c = k - 3 * tap, r = tap / 3, sx = tap - 3 * r;
        koff[ks][h2][e] = (k < 27) ? (c * PH + r) * PWP + sx + 1 : -1;
      }
  const bool vec_ok = (p.W % 4 == 0);
  const unsigned short* P = reinterpret_cast<const unsigned short*>(patch);
  uint8_t* wstage = stage + warp * 32 * PITCH;

  // Input patch items of this thread: item = (channel-row rc, group q); q == 0 is the single leading
  // column, q >= 1 a 16-byte group of four.  The next tile's items are fetched into registers before the
  // current tile is computed, so the global-load latency overlaps the gather / MMA / store of this tile.
  constexpr int NITEM = (3 * PH * 17 + 255) / 256;
  float4 pre[NITEM];
  auto fetch = [&](int tile) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int hi0 = 2 * th * TH - 1, wi0 = 2 * tw * TW - 1;  // wi0 + 1 is a multiple of 64: 16-byte aligned groups
#pragma unroll
    for (int it = 0; it < NITEM; ++it) {
      const int item = threadIdx.x + it * 256;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (item < 3 * PH * 17) {
        const int rc = item / 17, q = item - rc * 17;
        const int row = rc % PH, c = rc / PH;
        const int hi = hi0 + row;
        if (hi >= 0 && hi < p.H) {
          const int64_t rbase = (((int64_t)n * 3 + c) * p.H + hi) * p.W;
          if (q == 0) {
            if (wi0 >= 0)
              v.x = p.x_u8 ? (float)__ldg(reinterpret_cast<const uint8_t*>(p.x) + rbase + wi0) * p.in_scale
                           : __ldg(reinterpret_cast<const float*>(p.x) + rbase + wi0);
          } else {
            const int wi = wi0 + 1 + 4 * (q - 1);
            if (vec_ok && wi + 3 < p.W) {
              if (p.x_u8) {
                const uchar4 u = __ldg(reinterpret_cast<const uchar4*>(reinterpret_cast<const uint8_t*>(p.x) + rbase + wi));
                v = make_float4(u.x * p.in_scale, u.y * p.in_scale, u.z * p.in_scale, u.w * p.in_scale);
              } else {
                v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.x) + rbase + wi));
              }
            } else {
              float e[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
              for (int j = 0; j < 4; ++j)
                if (wi + j < p.W)
                  e[j] = p.x_u8 ? (float)__ldg(reinterpret_cast<const uint8_t*>(p.x) + rbase + wi + j) * p.in_scale
                                : __ldg(reinterpret_cast<const float*>(p.x) + rbase + wi + j);
              v = make_float4(e[0], e[1], e[2], e[3]);
            }
          }
        }
      }
      pre[it] = v;
    }
  };
  if ((int)blockIdx.x < num_tiles) fetch(blockIdx.x);

  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int px0 = tw * TW, py0 = th * TH;
    __syncthreads();                                       // previous tile's gathers are done with `patch`
#pragma unroll
    for (int it = 0; it < NITEM; ++it) {
      const int item = threadIdx.x + it * 256;
      if (item < 3 * PH * 17) {
        const int rc = item / 17, q = item - rc * 17;
        T* dst = patch + rc * PWP;
        if (q == 0) {
          dst[1] = T(pre[it].x);
        } else {
          uint32_t* d2 = reinterpret_cast<uint32_t*>(dst + 2 + 4 * (q - 1));
          d2[0] = stem_pack2<T>(pre[it].x, pre[it].y);
          d2[1] = stem_pack2<T>(pre[it].z, pre[it].w);
        }
      }
    }
    __syncthreads();
    if (tile + (int)gridDim.x < num_tiles) fetch(tile + gridDim.x);   // in flight during this tile's math
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mt][nt][j] = 0.f;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int base0 = (2 * warp) * PWP + 2 * (mt * 16 + g), base1 = base0 + 16;   // pixels g and g + 8
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t a[4];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int o0 = koff[ks][h2][0], o1 = koff[ks][h2][1];
          const uint32_t lo0 = o0 >= 0 ? P[base0 + o0] : 0u, hi0v = o1 >= 0 ? P[base0 + o1] : 0u;
          const uint32_t lo1 = o0 >= 0 ? P[base1 + o0] : 0u, hi1v = o1 >= 0 ? P[base1 + o1] : 0u;
          a[2 * h2 + 0] = lo0 | (hi0v << 16);
          a[2 * h2 + 1] = lo1 | (hi1v << 16);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) stem_mma16816<T>(acc[mt][nt], a, bfrag[nt][ks][0], bfrag[nt][ks][1]);
      }
    }
    // ---- bias + activation -> staged row of this warp -> coalesced 16-byte stores ----
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const float v0 = act_apply(acc[mt][nt][0] + bias[nt][0], p.act), v1 = act_apply(acc[mt][nt][1] + bias[nt][1], p.act);
        const float v2 = act_apply(acc[mt][nt][2] + bias[nt][0], p.act), v3 = act_apply(acc[mt][nt][3] + bias[nt][1], p.act);
        *reinterpret_cast<uint32_t*>(wstage + (mt * 16 + g) * PITCH + (nt * 8 + 2 * t) * 2) = stem_pack2<T>(v0, v1);
        *reinterpret_cast<uint32_t*>(wstage + (mt * 16 + g + 8) * PITCH + (nt * 8 + 2 * t) * 2) = stem_pack2<T>(v2, v3);
      }
    __syncwarp();
    const int py = py0 + warp;
    if (py < p.Ho) {
      const int valid = min(TW, p.Wo - px0);
      __nv_bfloat16* dst = p.y + (((int64_t)n * p.Ho + py) * p.Wo + px0) * COUT;
      constexpr int CPP = COUT / 8;                          // 16-byte chunks per pixel
      for (int i = lane; i < valid * CPP; i += 32) {
        const int px = i / CPP, part = i - px * CPP;
        reinterpret_cast<uint4*>(dst)[i] = *reinterpret_cast<const uint4*>(wstage + px * PITCH + part * 16);
      }
    }
    __syncwarp();
  }
}

template <int COUT>
__global__ void __launch_bounds__(256, 2) stem_mma_kernel(const StemParams p) {
  stem_mma_body<COUT, __nv_bfloat16>(p);
}
// fp16 activations (yv6_stem_fwd_f16)
template <int COUT>
__global__ void __launch_bounds__(256, 2) stem_mma_f16_kernel(const StemParams p) {
  stem_mma_body<COUT, __half>(p);
}

// fp32 images, asynchronous variant: the register prefetch above keeps 13 KB per CTA (26 KB per SM) of loads in flight, ~60 % of
// what HBM latency x bandwidth asks for (the kernel ran at 2.6 of 6.5 TB/s).  Here the input patch of a tile is copied global ->
// shared with cp.async (16-byte groups, zero fill outside the image) into a ring of three fp32 patches; two tiles are always in
// flight per CTA (56 KB per SM at two resident CTAs) and no register holds prefetched data.  The A fragments are gathered from the
// fp32 patch and rounded to bf16 on the way (cvt.rn.bf16x2), everything downstream is the kernel above.
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ACT = the layer's activation (YV6_ACT_*) at compile time: a runtime act_apply in the epilogue costs an indirect branch per
// element, and its SiLU / sigmoid divisions bring a CALL that pins the register allocation of every instance.  T: the activation
// dtype (the body of stem_mma_async_kernel and stem_mma_async_f16_kernel below).
template <int COUT, int ACT, typename T>
__device__ __forceinline__ void stem_mma_async_body(const StemParams& p) {
  constexpr int TH = 8, TW = 32, PH = 2 * TH + 1, NT = COUT / 8;
  constexpr int PWP = 72;                                  // fp32 patch row pitch; element j = input column 64 * tw + j - 4
  constexpr int PATCH = 3 * PH * PWP;                      // floats per stage
  constexpr int STAGES = 3;
  constexpr int PITCH = COUT * 2 + 16;
  extern __shared__ __align__(16) uint8_t stem_smem[];
  float* ring = reinterpret_cast<float*>(stem_smem);
  uint8_t* stage = stem_smem + (size_t)STAGES * PATCH * sizeof(float);
  const int tiles_w = (p.Wo + TW - 1) / TW, tiles_h = (p.Ho + TH - 1) / TH;
  const int num_tiles = tiles_w * tiles_h * p.N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;

  uint32_t bfrag[NT][2][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int k = ks * 16 + h2 * 8 + 2 * t, nn = nt * 8 + g;
        const float w0 = (k < 27) ? __ldg(p.w + k * COUT + nn) : 0.f;
        const float w1 = (k + 1 < 27) ? __ldg(p.w + (k + 1) * COUT + nn) : 0.f;
        bfrag[nt][ks][h2] = stem_pack2<T>(w0, w1);
      }
  float bias[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bias[nt][0] = p.b ? __ldg(p.b + nt * 8 + 2 * t) : 0.f;
    bias[nt][1] = p.b ? __ldg(p.b + nt * 8 + 2 * t + 1) : 0.f;
  }
  int koff[2][2][2];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = ks * 16 + h2 * 8 + 2 * t + e;
        const int tap = k / 3, c = k - 3 * tap, r = tap / 3, sx = tap - 3 * r;
        koff[ks][h2][e] = (k < 27) ? (c * PH + r) * PWP + sx + 3 : -1;   // input column 64 tw + 2 px + sx - 1 -> element 2 px + sx + 3
      }
  uint8_t* wstage = stage + warp * 32 * PITCH;
  const float* X = reinterpret_cast<const float*>(p.x);

  auto issue = [&](int tile, int slot) {     // one commit group per tile (possibly empty past the end: keeps the group count uniform)
    if (tile < num_tiles) {
      const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
      const int hi0 = 2 * th * TH - 1, wc0 = 64 * tw;      // first 16-byte group starts at input column 64 tw
      float* dst0 = ring + (size_t)slot * PATCH;
      for (int item = threadIdx.x; item < 3 * PH * 17; item += 256) {
        const int rc = item / 17, q = item - rc * 17;
        const int row = rc % PH, c = rc / PH;
        const int hi = hi0 + row;
        const bool row_ok = (hi >= 0 && hi < p.H);
        const float* src_row = X + (((int64_t)n * 3 + c) * p.H + (row_ok ? hi : 0)) * p.W;
        float* d = dst0 + rc * PWP;
        if (q == 0) {                                        // the single column left of the first group
          const int col = wc0 - 1;
          const bool ok = row_ok && col >= 0;
          cp_async4(d + 3, src_row + (ok ? col : 0), ok ? 4 : 0);
        } else {
          const int col = wc0 + 4 * (q - 1);
          const int nb = row_ok ? max(0, min(16, (p.W - col) * 4)) : 0;
          cp_async16(d + 4 + 4 * (q - 1), src_row + (nb > 0 ? col : 0), nb);
        }
      }
    }
    cp_async_commit();
  };
  issue(blockIdx.x, 0);
  issue(blockIdx.x + gridDim.x, 1);
  int slot = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int px0 = tw * TW, py0 = th * TH;
    cp_async_wait<1>();                                    // this tile's patch has landed (the next one may still be in flight)
    __syncthreads();                                       // ... for every thread's copies; the slot refilled below was read last iteration
    issue(tile + 2 * gridDim.x, (slot + 2) % STAGES);
    const float* P = ring + (size_t)slot * PATCH;
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mt][nt][j] = 0.f;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int base0 = (2 * warp) * PWP + 2 * (mt * 16 + g), base1 = base0 + 16;   // pixels g and g + 8
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t a[4];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int o0 = koff[ks][h2][0], o1 = koff[ks][h2][1];
          const float l0 = o0 >= 0 ? P[base0 + o0] : 0.f, h0 = o1 >= 0 ? P[base0 + o1] : 0.f;
          const float l1 = o0 >= 0 ? P[base1 + o0] : 0.f, h1 = o1 >= 0 ? P[base1 + o1] : 0.f;
          a[2 * h2 + 0] = stem_pack2<T>(l0, h0);
          a[2 * h2 + 1] = stem_pack2<T>(l1, h1);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) stem_mma16816<T>(acc[mt][nt], a, bfrag[nt][ks][0], bfrag[nt][ks][1]);
      }
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const float v0 = act_apply(acc[mt][nt][0] + bias[nt][0], ACT), v1 = act_apply(acc[mt][nt][1] + bias[nt][1], ACT);
        const float v2 = act_apply(acc[mt][nt][2] + bias[nt][0], ACT), v3 = act_apply(acc[mt][nt][3] + bias[nt][1], ACT);
        *reinterpret_cast<uint32_t*>(wstage + (mt * 16 + g) * PITCH + (nt * 8 + 2 * t) * 2) = stem_pack2<T>(v0, v1);
        *reinterpret_cast<uint32_t*>(wstage + (mt * 16 + g + 8) * PITCH + (nt * 8 + 2 * t) * 2) = stem_pack2<T>(v2, v3);
      }
    __syncwarp();
    const int py = py0 + warp;
    if (py < p.Ho) {
      const int valid = min(TW, p.Wo - px0);
      __nv_bfloat16* dst = p.y + (((int64_t)n * p.Ho + py) * p.Wo + px0) * COUT;
      constexpr int CPP = COUT / 8;
      for (int i = lane; i < valid * CPP; i += 32) {
        const int px = i / CPP, part = i - px * CPP;
        reinterpret_cast<uint4*>(dst)[i] = *reinterpret_cast<const uint4*>(wstage + px * PITCH + part * 16);
      }
    }
    __syncwarp();
    slot = (slot + 1) % STAGES;
  }
  cp_async_wait<0>();
}

template <int COUT, int ACT>
__global__ void __launch_bounds__(256, 2) stem_mma_async_kernel(const StemParams p) {
  stem_mma_async_body<COUT, ACT, __nv_bfloat16>(p);
}
template <int COUT, int ACT>
__global__ void __launch_bounds__(256, 2) stem_mma_async_f16_kernel(const StemParams p) {
  stem_mma_async_body<COUT, ACT, __half>(p);
}

// ------------------------------------------------------------------------------------------------
// SPPF pooling: reference SPPFModule / CSPSPPFModule (common.py:106-112, 150-158):
//   y1 = pool5(x), y2 = pool5(y1), y3 = pool5(y2), cat([x, y1, y2, y3]).
// With -inf padding the chained pools equal 5x5 / 9x9 / 13x13 windows clipped to the image.  One block
// = one image x 8 channels: the HxW plane is loaded into shared memory once, row maxima of the three
// window sizes are formed separably, then column maxima; results go to slices 1..3 of the concat buffer.
// ------------------------------------------------------------------------------------------------
struct PoolParams {
  __nv_bfloat16* buf;  // [planes][N,H,W,c_total] (fp16 for sppf_pool_f16_kernel, which only moves and compares its 16-bit values)
  int64_t plane_stride;
  int32_t N, H, W, C, c_total, planes;
};

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const __nv_bfloat162 b2 = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
    v[2 * j] = __low2float(b2);
    v[2 * j + 1] = __high2float(b2);
  }
}

__global__ void __launch_bounds__(256) sppf_pool_kernel(const PoolParams p) {
  extern __shared__ float sp[];                 // [4][H*W][8]: x, rowmax5, rowmax9, rowmax13
  const int cgs = p.C / 8;
  const int n = blockIdx.x / cgs, cg = blockIdx.x % cgs;
  const int HW = p.H * p.W;
  float* sx = sp;
  float* r5 = sp + (size_t)HW * 8;
  float* r9 = r5 + (size_t)HW * 8;
  float* r13 = r9 + (size_t)HW * 8;
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {
    const int64_t off = ((int64_t)n * HW + i) * p.c_total + cg * 8;
    float v[8];
    load8(p.buf + off, v);
    for (int pl = 1; pl < p.planes; ++pl) {
      float t[8];
      load8(p.buf + pl * p.plane_stride + off, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += t[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sx[i * 8 + j] = v[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {   // horizontal maxima
    const int h = i / p.W, w = i % p.W;
    float m5[8], m9[8], m13[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m5[j] = m9[j] = m13[j] = -INFINITY;
    for (int dx = -6; dx <= 6; ++dx) {
      const int ww = w + dx;
      if (ww < 0 || ww >= p.W) continue;
      const float* v = &sx[(h * p.W + ww) * 8];
      const int ad = abs(dx);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        m13[j] = fmaxf(m13[j], v[j]);
        if (ad <= 4) m9[j] = fmaxf(m9[j], v[j]);
        if (ad <= 2) m5[j] = fmaxf(m5[j], v[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { r5[i * 8 + j] = m5[j]; r9[i * 8 + j] = m9[j]; r13[i * 8 + j] = m13[j]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < HW; i += blockDim.x) {   // vertical maxima of the row maxima, then store
    const int h = i / p.W, w = i % p.W;
    float m[3][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[0][j] = m[1][j] = m[2][j] = -INFINITY;
    for (int dy = -6; dy <= 6; ++dy) {
      const int hh = h + dy;
      if (hh < 0 || hh >= p.H) continue;
      const int o = (hh * p.W + w) * 8;
      const int ad = abs(dy);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        m[2][j] = fmaxf(m[2][j], r13[o + j]);
        if (ad <= 4) m[1][j] = fmaxf(m[1][j], r9[o + j]);
        if (ad <= 2) m[0][j] = fmaxf(m[0][j], r5[o + j]);
      }
    }
    const int64_t o = ((int64_t)n * HW + i) * p.c_total + cg * 8;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      for (int pl = 0; pl < p.planes; ++pl) {
        uint32_t wds[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          __nv_bfloat162 b2 = __floats2bfloat162_rn(m[k][2 * j], m[k][2 * j + 1]);
          wds[j] = *reinterpret_cast<uint32_t*>(&b2);
          m[k][2 * j] -= __low2float(b2);
          m[k][2 * j + 1] -= __high2float(b2);
        }
        *reinterpret_cast<uint4*>(p.buf + pl * p.plane_stride + o + (int64_t)(k + 1) * p.C) =
            make_uint4(wds[0], wds[1], wds[2], wds[3]);
      }
    }
  }
}

// bf16 (single plane) variant: a maximum of bf16 values is itself one of them, so the whole pyramid runs on packed
// bf16x2 values with no rounding anywhere -- bit-identical to the fp32 kernel above.  One CTA per (image, 16 channels):
// a pixel's 32 bytes are one full DRAM sector (the fp32 kernel's 8-channel slices fetched half-used sectors at a 2 KB
// stride: 0.6 TB/s), the staged plane and its three row-maximum planes take 4 x H*W*32 bytes of shared memory.
// The same holds for fp16 (half2 maxima): T2 = __nv_bfloat162 or __half2.
template <typename T2>
__device__ __forceinline__ uint4 hmax8(uint4 a, uint4 b) {
  uint4 r;
  *reinterpret_cast<T2*>(&r.x) = __hmax2(*reinterpret_cast<T2*>(&a.x), *reinterpret_cast<T2*>(&b.x));
  *reinterpret_cast<T2*>(&r.y) = __hmax2(*reinterpret_cast<T2*>(&a.y), *reinterpret_cast<T2*>(&b.y));
  *reinterpret_cast<T2*>(&r.z) = __hmax2(*reinterpret_cast<T2*>(&a.z), *reinterpret_cast<T2*>(&b.z));
  *reinterpret_cast<T2*>(&r.w) = __hmax2(*reinterpret_cast<T2*>(&a.w), *reinterpret_cast<T2*>(&b.w));
  return r;
}

template <typename T2>
__device__ __forceinline__ void sppf_pool_packed_body(const PoolParams& p) {
  extern __shared__ uint4 sq[];                 // [4][H*W][2] units of 8 channels: x, rowmax5, rowmax9, rowmax13
  const int cgs = p.C / 16;
  const int n = blockIdx.x / cgs, cg = blockIdx.x % cgs;
  const int HW = p.H * p.W, U = HW * 2;
  uint4* sx = sq;
  uint4* r5 = sq + U;
  uint4* r9 = r5 + U;
  uint4* r13 = r9 + U;
  const __nv_bfloat16* src = p.buf + (int64_t)n * HW * p.c_total + cg * 16;
  for (int u = threadIdx.x; u < U; u += blockDim.x)      // two adjacent threads fetch one pixel's 32-byte sector
    sx[u] = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(u >> 1) * p.c_total + (u & 1) * 8));
  __syncthreads();
  for (int u = threadIdx.x; u < U; u += blockDim.x) {    // horizontal maxima over 5 / 9 / 13 columns (clipped at the border)
    const int i = u >> 1, half = u & 1;
    const int h = i / p.W, w = i - h * p.W;
    uint4 m5 = sx[u], m9, m13;
#pragma unroll
    for (int dx = 1; dx <= 2; ++dx) {
      if (w - dx >= 0) m5 = hmax8<T2>(m5, sx[u - 2 * dx]);
      if (w + dx < p.W) m5 = hmax8<T2>(m5, sx[u + 2 * dx]);
    }
    m9 = m5;
#pragma unroll
    for (int dx = 3; dx <= 4; ++dx) {
      if (w - dx >= 0) m9 = hmax8<T2>(m9, sx[u - 2 * dx]);
      if (w + dx < p.W) m9 = hmax8<T2>(m9, sx[u + 2 * dx]);
    }
    m13 = m9;
#pragma unroll
    for (int dx = 5; dx <= 6; ++dx) {
      if (w - dx >= 0) m13 = hmax8<T2>(m13, sx[u - 2 * dx]);
      if (w + dx < p.W) m13 = hmax8<T2>(m13, sx[u + 2 * dx]);
    }
    (void)half;
    r5[u] = m5;
    r9[u] = m9;
    r13[u] = m13;
  }
  __syncthreads();
  __nv_bfloat16* dst = p.buf + (int64_t)n * HW * p.c_total + cg * 16;
  const int rs = 2 * p.W;                                // units per image row
  for (int u = threadIdx.x; u < U; u += blockDim.x) {    // vertical maxima of the row maxima, then store the three slices
    const int i = u >> 1;
    const int h = i / p.W;
    uint4 m5 = r5[u], m9 = r9[u], m13 = r13[u];
#pragma unroll
    for (int dy = 1; dy <= 6; ++dy) {
      if (h - dy >= 0) {
        if (dy <= 2) m5 = hmax8<T2>(m5, r5[u - dy * rs]);
        if (dy <= 4) m9 = hmax8<T2>(m9, r9[u - dy * rs]);
        m13 = hmax8<T2>(m13, r13[u - dy * rs]);
      }
      if (h + dy < p.H) {
        if (dy <= 2) m5 = hmax8<T2>(m5, r5[u + dy * rs]);
        if (dy <= 4) m9 = hmax8<T2>(m9, r9[u + dy * rs]);
        m13 = hmax8<T2>(m13, r13[u + dy * rs]);
      }
    }
    __nv_bfloat16* o = dst + (int64_t)i * p.c_total + (u & 1) * 8;
    *reinterpret_cast<uint4*>(o + (int64_t)p.C) = m5;
    *reinterpret_cast<uint4*>(o + (int64_t)2 * p.C) = m9;
    *reinterpret_cast<uint4*>(o + (int64_t)3 * p.C) = m13;
  }
}

__global__ void __launch_bounds__(256) sppf_pool_bf16_kernel(const PoolParams p) { sppf_pool_packed_body<__nv_bfloat162>(p); }
__global__ void __launch_bounds__(256) sppf_pool_f16_kernel(const PoolParams p) { sppf_pool_packed_body<__half2>(p); }

// ------------------------------------------------------------------------------------------------
// head decode: eval tail of Detect.forward (effidehead.py:106-139), generate_anchors(is_eval)
// (anchor_generator.py:13-33) and dist2bbox(xywh) (general.py:32-43).  One warp per anchor row:
// lanes stream the nc class scores (already sigmoid-ed by the cls_pred conv epilogue), lanes 0..3
// decode one box side each.  fp32 ops are explicit round-to-nearest (no FMA contraction) in the
// reference's order so that box bits match the reference's fp32 path.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxLevels = 6;
struct DecodeParams {
  const float* cls;  // [B, A, nc]
  const float* reg;  // [B, A, R]
  float* out;        // [B, A, 5 + nc]
  int32_t B, A, nc, R, reg_max, nl;
  int32_t lvl_off[kMaxLevels + 1];
  int32_t lvl_w[kMaxLevels];
  float lvl_stride[kMaxLevels];
};

__global__ void __launch_bounds__(256) head_decode_kernel(const __grid_constant__ DecodeParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= (int64_t)p.B * p.A) return;
  const int a = (int)(row % p.A);
  const float* cls = p.cls + row * p.nc;
  float* out = p.out + row * (5 + p.nc);
  for (int c = lane; c < p.nc; c += 32) out[5 + c] = __ldg(cls + c);
  // distances: plain ltrb (R == 4) or DFL expectation over reg_max+1 bins per side
  float dist = 0.f;
  if (lane < 4) {
    const float* reg = p.reg + row * p.R;
    if (p.R == 4) {
      dist = __ldg(reg + lane);
    } else {
      const int nb = p.reg_max + 1;
      const float* l = reg + lane * nb;
      float mx = -INFINITY;
      for (int i = 0; i < nb; ++i) mx = fmaxf(mx, __ldg(l + i));
      float den = 0.f;
      for (int i = 0; i < nb; ++i) den += expf(__ldg(l + i) - mx);
      float e = 0.f;
      for (int i = 0; i < nb; ++i) e = __fadd_rn(e, __fmul_rn(expf(__ldg(l + i) - mx) / den, (float)i));
      dist = e;
    }
  }
  const float dl = __shfl_sync(0xffffffffu, dist, 0), dt = __shfl_sync(0xffffffffu, dist, 1);
  const float dr = __shfl_sync(0xffffffffu, dist, 2), db = __shfl_sync(0xffffffffu, dist, 3);
  if (lane == 0) {
    int lvl = 0;
    while (lvl + 1 < p.nl && a >= p.lvl_off[lvl + 1]) ++lvl;
    const int local = a - p.lvl_off[lvl];
    const float ax = (float)(local % p.lvl_w[lvl]) + 0.5f;
    const float ay = (float)(local / p.lvl_w[lvl]) + 0.5f;
    const float s = p.lvl_stride[lvl];
    const float x1 = __fsub_rn(ax, dl), y1 = __fsub_rn(ay, dt);
    const float x2 = __fadd_rn(ax, dr), y2 = __fadd_rn(ay, db);
    out[0] = __fmul_rn(__fdiv_rn(__fadd_rn(x1, x2), 2.f), s);
    out[1] = __fmul_rn(__fdiv_rn(__fadd_rn(y1, y2), 2.f), s);
    out[2] = __fmul_rn(__fsub_rn(x2, x1), s);
    out[3] = __fmul_rn(__fsub_rn(y2, y1), s);
    out[4] = 1.0f;
  }
}

}  // namespace yv6

using namespace yv6;

using StemKernelFn = void (*)(const StemParams);
#define YV6_STEM_ACTS(K, C)                                                                                          \
  {K<C, YV6_ACT_NONE>, K<C, YV6_ACT_RELU>, K<C, YV6_ACT_SILU>, K<C, YV6_ACT_SIGMOID>, K<C, YV6_ACT_HARDSWISH>, \
   K<C, YV6_ACT_HARDSIGMOID>}
#define YV6_STEM_TABLE(K) {YV6_STEM_ACTS(K, 16), YV6_STEM_ACTS(K, 32), YV6_STEM_ACTS(K, 48), YV6_STEM_ACTS(K, 64)}
// [fp16 output][Cout / 16 - 1][act]
static const StemKernelFn kStemAsync[2][4][6] = {YV6_STEM_TABLE(stem_mma_async_kernel), YV6_STEM_TABLE(stem_mma_async_f16_kernel)};
#undef YV6_STEM_TABLE
#undef YV6_STEM_ACTS
// [fp16 output][Cout / 16 - 1]
static const StemKernelFn kStemSync[2][4] = {{stem_mma_kernel<16>, stem_mma_kernel<32>, stem_mma_kernel<48>, stem_mma_kernel<64>},
                                             {stem_mma_f16_kernel<16>, stem_mma_f16_kernel<32>, stem_mma_f16_kernel<48>,
                                              stem_mma_f16_kernel<64>}};

static int stem_fwd(yv6_handle* h, const yv6_stem_desc* d, void* stream, bool f16) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->x && d->w && d->y, "stem: null argument");
  YV6_REQUIRE(!f16 || (d->nsplit == 1 && !d->fp32_math), "stem_f16: nsplit must be 1 and fp32_math 0");
  YV6_REQUIRE(d->Cout > 0 && d->Cout <= kStemMaxCout && d->Cout % 16 == 0, "stem: Cout=%d must be 16/32/48/64", d->Cout);
  YV6_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "stem: nsplit must be 1 or 3");
  YV6_REQUIRE(d->x_dtype == YV6_DT_F32 || d->x_dtype == YV6_DT_U8, "stem: image must be fp32 or uint8");
  StemParams p;
  p.w = d->w;
  p.b = d->bias;
  p.x = d->x;
  p.y = reinterpret_cast<__nv_bfloat16*>(d->y);
  p.y_plane_stride = d->y_plane_stride;
  p.N = d->N;
  p.H = d->H;
  p.W = d->W;
  p.Ho = (d->H + 2 - 3) / 2 + 1;
  p.Wo = (d->W + 2 - 3) / 2 + 1;
  p.x_u8 = (d->x_dtype == YV6_DT_U8);
  p.in_scale = d->in_scale;
  p.act = d->act;
  p.planes = d->nsplit;
  const int64_t total = (int64_t)p.N * p.Ho * p.Wo;
  const unsigned grid = (unsigned)((total + 255) / 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (d->nsplit == 1 && !d->fp32_math) {
    // bf16 activations: tensor-core path (bf16 image / weights, fp32 accumulate)
    const unsigned ntile = (unsigned)(((p.Wo + 31) / 32) * ((p.Ho + 7) / 8) * p.N);
    const unsigned tiles = std::min<unsigned>(ntile, (unsigned)h->num_sms * 2);   // persistent CTAs, two resident per SM (register budget)
    // fp32 images whose rows are 16-byte aligned: asynchronous shared-memory ring (3 x 14.7 KB patches + the output staging)
    if (!p.x_u8 && p.W % 4 == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && (d->Cout == 16 || d->Cout == 32 || d->Cout == 48 || d->Cout == 64) &&
        d->force_sync_loads == 0) {
      const size_t smem = (size_t)3 * 3 * 17 * 72 * 4 + (size_t)8 * 32 * (d->Cout * 2 + 16);
      if (!(h->configured & YV6_CFG_STEM)) {
        for (const auto& by_dtype : kStemAsync)
          for (const auto& by_act : by_dtype)
            for (StemKernelFn fn : by_act) YV6_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        h->configured |= YV6_CFG_STEM;
      }
      // act_apply treats codes outside the enum as no activation
      const int act = (d->act >= YV6_ACT_NONE && d->act <= YV6_ACT_HARDSIGMOID) ? d->act : YV6_ACT_NONE;
      kStemAsync[f16][d->Cout / 16 - 1][act]<<<tiles, 256, smem, s>>>(p);
      YV6_CHECK_CUDA(cudaGetLastError());
      return YV6_OK;
    }
    kStemSync[f16][d->Cout / 16 - 1]<<<tiles, 256, 0, s>>>(p);
    YV6_CHECK_CUDA(cudaGetLastError());
    return YV6_OK;
  }
  switch (d->Cout) {
    case 16: stem_kernel<16><<<grid, 256, 0, s>>>(p); break;
    case 32: stem_kernel<32><<<grid, 256, 0, s>>>(p); break;
    case 48: stem_kernel<48><<<grid, 256, 0, s>>>(p); break;
    default: stem_kernel<64><<<grid, 256, 0, s>>>(p); break;
  }
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_stem_fwd(yv6_handle* h, const yv6_stem_desc* d, void* stream) { return stem_fwd(h, d, stream, false); }
extern "C" int yv6_stem_fwd_f16(yv6_handle* h, const yv6_stem_desc* d, void* stream) { return stem_fwd(h, d, stream, true); }

extern "C" int yv6_sppf_pool_f16(yv6_handle* h, void* buf, int32_t N, int32_t H, int32_t W, int32_t C, int32_t c_total,
                                 int32_t nsplit, int64_t plane_stride, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && buf, "sppf_pool_f16: null argument");
  YV6_REQUIRE(nsplit == 1, "sppf_pool_f16: nsplit must be 1");
  YV6_REQUIRE(C % 16 == 0 && c_total >= 4 * C && c_total % 8 == 0, "sppf_pool_f16: bad channels C=%d c_total=%d", C, c_total);
  const size_t smem16 = (size_t)4 * H * W * 32;
  YV6_REQUIRE(smem16 <= (size_t)h->max_smem_optin, "sppf_pool_f16: %dx%d plane does not fit in shared memory", H, W);
  (void)plane_stride;                                    // one plane
  PoolParams p{reinterpret_cast<__nv_bfloat16*>(buf), 0, N, H, W, C, c_total, 1};
  if (!(h->configured & YV6_CFG_POOLF16)) {
    YV6_CHECK_CUDA(cudaFuncSetAttribute(sppf_pool_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->max_smem_optin));
    h->configured |= YV6_CFG_POOLF16;
  }
  sppf_pool_f16_kernel<<<(unsigned)(N * (C / 16)), 256, smem16, (cudaStream_t)stream>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_sppf_pool(yv6_handle* h, void* buf, int32_t N, int32_t H, int32_t W, int32_t C, int32_t c_total,
                             int32_t nsplit, int64_t plane_stride, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && buf, "sppf_pool: null argument");
  YV6_REQUIRE(C % 8 == 0 && c_total >= 4 * C && c_total % 8 == 0, "sppf_pool: bad channels C=%d c_total=%d", C, c_total);
  const size_t smem = (size_t)4 * H * W * 8 * sizeof(float);
  YV6_REQUIRE(smem <= (size_t)h->max_smem_optin, "sppf_pool: %dx%d plane does not fit in shared memory", H, W);
  PoolParams p{reinterpret_cast<__nv_bfloat16*>(buf), plane_stride, N, H, W, C, c_total, nsplit == 3 ? 3 : 1};
  if (!(h->configured & YV6_CFG_POOL)) {
    YV6_CHECK_CUDA(cudaFuncSetAttribute(sppf_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->max_smem_optin));
    h->configured |= YV6_CFG_POOL;
  }
  const size_t smem16 = (size_t)4 * H * W * 32;
  if (nsplit != 3 && C % 16 == 0 && smem16 <= (size_t)h->max_smem_optin) {   // bf16 activations: packed, sector-sized channel slices
    if (!(h->configured & YV6_CFG_POOL16)) {
      YV6_CHECK_CUDA(cudaFuncSetAttribute(sppf_pool_bf16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->max_smem_optin));
      h->configured |= YV6_CFG_POOL16;
    }
    sppf_pool_bf16_kernel<<<(unsigned)(N * (C / 16)), 256, smem16, (cudaStream_t)stream>>>(p);
    YV6_CHECK_CUDA(cudaGetLastError());
    return YV6_OK;
  }
  sppf_pool_kernel<<<(unsigned)(N * (C / 8)), 256, smem, (cudaStream_t)stream>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_head_decode(yv6_handle* h, const float* cls, const float* reg, float* out, int32_t B, int32_t nc,
                               int32_t reg_ch, int32_t nl, const int32_t* lvl_h, const int32_t* lvl_w,
                               const float* lvl_stride, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && cls && reg && out && lvl_h && lvl_w && lvl_stride, "head_decode: null argument");
  YV6_REQUIRE(nl >= 1 && nl <= kMaxLevels, "head_decode: nl=%d out of range", nl);
  YV6_REQUIRE(reg_ch == 4 || reg_ch % 4 == 0, "head_decode: reg_ch=%d", reg_ch);
  DecodeParams p;
  p.cls = cls;
  p.reg = reg;
  p.out = out;
  p.B = B;
  p.nc = nc;
  p.R = reg_ch;
  p.reg_max = reg_ch / 4 - 1;
  p.nl = nl;
  int off = 0;
  for (int l = 0; l < nl; ++l) {
    p.lvl_off[l] = off;
    p.lvl_w[l] = lvl_w[l];
    p.lvl_stride[l] = lvl_stride[l];
    off += lvl_h[l] * lvl_w[l];
  }
  p.lvl_off[nl] = off;
  p.A = off;
  const int64_t rows = (int64_t)B * p.A;
  head_decode_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
