// yv6_conv_igemm.cu -- fused implicit-GEMM convolution on Hopper warpgroup tensor cores (wgmma, sm_90a).
//
// Computes, for NHWC bf16 activations and KRSC bf16 weights,
//     y = act(conv(x, w) + bias) [+ alpha * residual]
// which in deploy form is every 3x3 / 1x1 conv of the YOLOv6 backbones, necks and head:
// ConvModule.forward_fuse (reference yolov6/layers/common.py:50-54), RepVGGBlock with
// rbr_reparam (common.py:247-248), BottleRep's shortcut (common.py:605-608), the 1x1s of
// BiFusion/BepC3/CSPSPPF, the head stems and preds (effidehead.py:72-118) and, through the
// output strides, torch.cat (reppan.py:228,232) and ConvTranspose2d k2s2 (common.py:181-194).
//
// Design (im2col-free):
//   * GEMM view: M = output pixels, N = Cout, K = taps x Cin.  One M tile is a BW x BH x BI box of
//     output pixels (<= 128 rows).  For filter tap (r,s) the A tile is that same box of the INPUT
//     shifted by (r-pad, s-pad): one TMA box load from a 5-D tensor map (C, W, H, N, plane) with
//     zero fill out of bounds (= conv padding) and elementStrides = conv stride.  The box lands in
//     shared memory as `rows` consecutive K-major rows in the 128/64/32-byte swizzle that
//     wgmma consumes directly -- no im2col buffer, no index math on the SMs.
//   * B tile = [BN x KB] slice of the weights, one TMA load from a 3-D map (K, Cout, plane).
//   * warpgroup 0 = TMA producer (one warp), warpgroups 1 and 2 = consumers in a ping-pong schedule: each owns
//     every other tile of the CTA, issues wgmma m64nBNk16 for all 128 rows of it and keeps its accumulators in
//     registers.  The two take turns on the tensor cores, so one's epilogue runs under the other's MMAs.
//     The epilogue adds the bias and applies the activation in registers, stages the tile in the output dtype and
//     writes it with TMA bulk tensor stores through a third tensor map over the destination view (channel slice,
//     ConvTranspose quadrant, head anchors).  Residual adds, bf16x3 output planes and views no tensor map can describe
//     take the chunk epilogue: an fp32 staging tile written out in coalesced 16-channel chunks.
//   * persistent CTAs (grid = #SMs) over a static tile schedule; smem ring of `stages` K-blocks
//     (the producer runs ahead across tiles, so the next tile's loads overlap this tile's epilogue).
//   * bf16x3 mode (nsplit=3): same kernel, K loop additionally runs over six (plane_a, plane_b)
//     pairs, giving fp32-equivalent products with fp32 accumulation.
//   * halo variants (MODE 1 / 2: 3x3 stride 1; MODE 3 / 4: 3x3 stride 2 on the column-pair view of the input): ONE input box
//     per channel block feeds every tap through shifted wgmma descriptors; weights streamed through their own ring or resident.
//     At BN = 64 the tile is computed transposed, 64 channels x 128 pixels (mma_kblock_t): one m64n128k16 per k16 step.
//   * CTA-pair variants (CP = true): clusters of two CTAs on adjacent M tiles; each loads half of the weight tile with a TMA
//     multicast into both CTAs.
#include <algorithm>
#include <cstdarg>
#include <type_traits>

#include "yv6_common.cuh"
#include "yv6_handle.h"
#include "yv6_wgmma.cuh"

namespace yv6 {

constexpr int kConvThreads = 384;   // producer warpgroup + two consumer warpgroups
constexpr int kMaxStages = 12;
constexpr int kTileRows = 128;

struct ConvKParams {
  int32_t BW, BH, BI, rows;
  int32_t tiles_w, tiles_h, tiles_i, tiles_n, num_tiles;
  int32_t N, Ho, Wo, Cout, BN;
  int32_t taps, kw, stride, stride_w, pad, pad_w, Cin;   // stride / pad = rows (h), stride_w / pad_w = columns
  int32_t cin_blocks, kb_elems, kb_bytes, ksteps;
  int32_t sbo_bytes, layout_type;
  int32_t npairs;
  int32_t stages, a_stage_bytes, b_stage_bytes;
  int32_t act, y_dtype, out_planes, res_planes;
  void* y;
  int64_t y_img_stride, y_h_stride, y_w_stride, y_plane_stride;
  const void* res;          // the operand dtype (bf16 or fp16)
  float alpha;
  int64_t res_img_stride, res_h_stride, res_w_stride, res_plane_stride;
  const float* bias;
  // halo mode (3x3 stride-1, Cin % 64 == 0): one (BH+2)x(BW+2) input box per channel block feeds all
  // nine taps through wgmma descriptors offset into it; B tiles ride their own ring (or stay resident).
  int32_t halo, a_stages, b_stages, b_resident;   // halo: 1 = 3x3 stride 1, 2 = column-pair view of a 3x3 stride-2 conv
  int32_t skip_cb;                                // halo 2: the first skip_cb channel blocks of the s = 0 taps are all-zero weights (skipped)
  int32_t a_region_bytes, b_region_bytes;  // smem carve: [A ring][B ring][fp32 output tile][barriers]
  // CTA-pair mode (clusters of two CTAs): one schedule unit = two consecutive M tiles (one per CTA) x one N tile.  Each CTA
  // loads HALF of the weight tile (b_rows = BN / 2 rows) and multicasts it into both CTAs, so every weight byte crosses from
  // L2 once per pair instead of once per CTA.  A ring stage may only be refilled once the consumers of BOTH CTAs released it.
  int32_t cpair, m_tiles, b_rows;
  int32_t fast_act;                        // bf16 outputs: SiLU through tanh.approx (rel. error 2^-11 < bf16 ulp)
  // 1: the epilogue writes the tile through the output tensor map tmY (conditions in plan_conv); 0: in 16-channel chunks
  int32_t tma_store;
};

constexpr int kHaloW = 10, kHaloH = 18;                   // BW = 8, BH = 16 output tile + 1-pixel border
// Halo geometry of a kernel variant.  S2 = false: 3x3 stride 1 (above).  S2 = true: 3x2 kernel with stride (2, 1) and padding
// (1, 1) -- a 3x3 stride-2 conv on the column-pair view [N, H, W/2, 2C] of its input: the same 8 x 16 output tile reads a
// 9 x 33 box; tap (r, s) starts (9 r + s) pixels into it and consecutive output rows are TWO box rows apart (the wgmma
// descriptor's stride between 8-row groups), so the stride costs nothing at issue time.
template <bool S2>
struct HaloGeom {
  static constexpr int W = S2 ? 9 : kHaloW, H = S2 ? 33 : kHaloH, KW = S2 ? 2 : 3, TAPS = S2 ? 6 : 9, SH = S2 ? 2 : 1;
  static constexpr int kBytes = W * H * 128;
  static constexpr int kStageBytes = ((kBytes + 1023) / 1024) * 1024;     // 24 KB / 38 KB
};
constexpr int kMaxAStages = 6, kMaxBStages = 40;

// fp32 staging tile of the epilogue: 128 rows x BN columns, rows padded by 4 floats (16-byte aligned, fewer bank conflicts);
// each consumer warpgroup owns 64 of the rows and writes its tile out through them in two passes.  The TMA-store epilogue
// uses the same half differently: its first 256 x BN bytes hold the whole tile in bf16 (or 64 rows of it in fp32) for the
// bulk tensor store, the 1 KB after them the tile's bias.
__host__ __device__ constexpr int stage_pitch(int bn) { return bn + 4; }
__host__ __device__ constexpr int staging_bytes(int bn) { return kTileRows * stage_pitch(bn) * 4; }
static_assert(staging_bytes(32) / 2 == 256 * 32 + 1024, "the TMA-store tile and its bias fill one staging half");

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// The same load delivered to the same shared-memory offset (and its bytes to the same barrier offset) in every CTA of
// `mask` within the cluster.
__device__ __forceinline__ void tma_load_3d_mc(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
      : "memory");
}
// Bulk tensor store of a shared-memory box to (c0, c1, c2, c3) of the output map (elements out of bounds are not written), in
// the issuing thread's bulk async-group.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the stores this thread committed have finished reading shared memory
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// this thread's shared-memory writes become visible to the async proxy (the TMA unit)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void warpgroup_bar_sync(int wg) {  // the 128 threads of consumer warpgroup wg (named barrier 1 + wg)
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}
// warp-specialised register split: the producer warpgroup gives registers back, the two consumer warpgroups take them
// (128 x 40 + 256 x 232 <= 64 K), so that a consumer can hold the fp32 accumulators of a whole 128 x BN tile
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

struct TileCoord {
  int w0, h0, i0, n0;
};
__device__ __forceinline__ TileCoord decode_tile(const ConvKParams& p, int tile) {
  TileCoord t;
  int nt = tile % p.tiles_n;
  int m = tile / p.tiles_n;
  int tw = m % p.tiles_w;
  m /= p.tiles_w;
  int th = m % p.tiles_h;
  int ti = m / p.tiles_h;
  t.w0 = tw * p.BW;
  t.h0 = th * p.BH;
  t.i0 = ti * p.BI;
  t.n0 = nt * p.BN;
  return t;
}

// CTA-pair mode: unit -> (M tile 2u + rank, N tile).  A missing second tile (odd tile count) is placed on image N: its TMA
// loads are zero filled and its stores dropped, so it needs no special case anywhere.
__device__ __forceinline__ TileCoord decode_unit(const ConvKParams& p, int unit, int rank) {
  TileCoord t;
  const int nt = unit % p.tiles_n;
  int m = (unit / p.tiles_n) * 2 + rank;
  t.n0 = nt * p.BN;
  if (m >= p.m_tiles) {
    t.w0 = 0;
    t.h0 = 0;
    t.i0 = p.N;
    return t;
  }
  const int tw = m % p.tiles_w;
  m /= p.tiles_w;
  const int th = m % p.tiles_h;
  const int ti = m / p.tiles_h;
  t.w0 = tw * p.BW;
  t.h0 = th * p.BH;
  t.i0 = ti * p.BI;
  return t;
}

// bf16x3 plane pairs, smallest products first; the plain bf16 mode uses the last entry only.
__constant__ int kPairA[6] = {0, 1, 2, 0, 1, 0};
__constant__ int kPairB[6] = {2, 1, 0, 1, 0, 0};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// The operand dtype T (__nv_bfloat16, or __half for the fp16 mode) of activations, weights and residuals: rounding to it,
// and its packed pair.  fp16 rounds values beyond 65504 to +-inf.
template <typename T> struct Pair2;
template <> struct Pair2<__nv_bfloat16> { using type = __nv_bfloat162; };
template <> struct Pair2<__half> { using type = __half2; };
template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (std::is_same_v<T, __half>) {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    return pack_bf16x2(a, b);
  }
}
template <typename T>
__device__ __forceinline__ T round_to(float v) {
  if constexpr (std::is_same_v<T, __half>) return __float2half_rn(v);
  else return __float2bfloat16_rn(v);
}
__device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }

// Store 16 consecutive output channels of one pixel.
template <typename T>
__device__ __forceinline__ void store_chunk(const ConvKParams& p, int64_t off, int n, int ncol,
                                            const float (&v)[16]) {
  if (p.y_dtype == YV6_DT_F32) {
    float* y = reinterpret_cast<float*>(p.y) + off + n;
    if (ncol == 16 && ((reinterpret_cast<uintptr_t>(y) & 15) == 0)) {
      float4* y4 = reinterpret_cast<float4*>(y);
#pragma unroll
      for (int j = 0; j < 4; ++j) y4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
      for (int j = 0; j < ncol; ++j) y[j] = v[j];
    }
    return;
  }
  float rem[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) rem[j] = v[j];
  for (int pl = 0; pl < p.out_planes; ++pl) {
    T* y = reinterpret_cast<T*>(p.y) + pl * p.y_plane_stride + off + n;
    if (ncol == 16 && ((reinterpret_cast<uintptr_t>(y) & 15) == 0)) {
      uint4 q0, q1;
      q0.x = pack2<T>(rem[0], rem[1]);
      q0.y = pack2<T>(rem[2], rem[3]);
      q0.z = pack2<T>(rem[4], rem[5]);
      q0.w = pack2<T>(rem[6], rem[7]);
      q1.x = pack2<T>(rem[8], rem[9]);
      q1.y = pack2<T>(rem[10], rem[11]);
      q1.z = pack2<T>(rem[12], rem[13]);
      q1.w = pack2<T>(rem[14], rem[15]);
      reinterpret_cast<uint4*>(y)[0] = q0;
      reinterpret_cast<uint4*>(y)[1] = q1;
    } else {
      for (int j = 0; j < ncol; ++j) y[j] = round_to<T>(rem[j]);
    }
    if (pl + 1 < p.out_planes) {
#pragma unroll
      for (int j = 0; j < 16; ++j) rem[j] -= to_float(round_to<T>(rem[j]));
    }
  }
}



__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// the layer's activation on n values (after the bias), shared by both epilogues so that they round alike
template <int N>
__device__ __forceinline__ void activate(const ConvKParams& p, float (&v)[N]) {
  if (p.act == YV6_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = fmaxf(v[j], 0.f);
  } else if (p.act == YV6_ACT_SILU) {
    if (p.fast_act) {                       // x * sigmoid(x) = h + h * tanh(h), h = x / 2: one MUFU per element
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const float h = 0.5f * v[j];
        v[j] = fmaf(h, tanh_fast(h), h);
      }
    } else {                                // ex2 / rcp approximations are ~1e-7 relative
#pragma unroll
      for (int j = 0; j < N; ++j) v[j] = v[j] * rcp_ftz(1.f + ex2_ftz(-1.4426950408889634f * v[j]));
    }
  } else if (p.act == YV6_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = rcp_ftz(1.f + ex2_ftz(-1.4426950408889634f * v[j]));
  } else if (p.act == YV6_ACT_HARDSWISH) {  // the YOLOv6Lite ConvBNHS convs
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = v[j] * fminf(fmaxf(v[j] + 3.f, 0.f), 6.f) * (1.f / 6.f);   // no division: it would bring a CALL
  }
}

// bias + activation (+ residual) for 16 consecutive output channels of one pixel
template <typename T>
__device__ __forceinline__ void epilogue_math(const ConvKParams& p, const uint32_t (&r)[16], int n, int ncol, int64_t roff,
                                              float (&v)[16]) {
  if (p.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n) + j);
      v[4 * j + 0] = __uint_as_float(r[4 * j + 0]) + b.x;
      v[4 * j + 1] = __uint_as_float(r[4 * j + 1]) + b.y;
      v[4 * j + 2] = __uint_as_float(r[4 * j + 2]) + b.z;
      v[4 * j + 3] = __uint_as_float(r[4 * j + 3]) + b.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(r[j]);
  }
  activate(p, v);
  if (p.res != nullptr) {
    for (int pl = 0; pl < p.res_planes; ++pl) {
      const T* rp = reinterpret_cast<const T*>(p.res) + pl * p.res_plane_stride + roff + n;
      if (ncol == 16 && ((reinterpret_cast<uintptr_t>(rp) & 15) == 0)) {
        const uint4 q0 = __ldg(reinterpret_cast<const uint4*>(rp));
        const uint4 q1 = __ldg(reinterpret_cast<const uint4*>(rp) + 1);
        const uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const typename Pair2<T>::type b2 = *reinterpret_cast<const typename Pair2<T>::type*>(&w[j]);
          v[2 * j] += p.alpha * __low2float(b2);
          v[2 * j + 1] += p.alpha * __high2float(b2);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < ncol) v[j] += p.alpha * to_float(rp[j]);
      }
    }
  }
}

// TMA-store epilogue: the output box is (y_box_bytes / element size) channels x the output tile, and its rows are y_box_bytes
// long, which is also the swizzle span of the map (the widest of 128 / 64 bytes that divides a BN-wide row)
__host__ __device__ constexpr int y_box_bytes(int bn, int esz) { return (bn * esz) % 128 == 0 ? 128 : 64; }

// TMA-store epilogue: bias + activation on one accumulator half (rows row0 + 8 i, columns 8 j + c0, + 1 of this thread), rounded
// to the output dtype and written to the staging half as the boxes of the output map: column group g (kCols channels) is a
// [rows][kBox bytes] block at g * kGroupBytes in the map's swizzle, which XORs the 16-byte unit of a row with address bits 7+.
template <typename T, int BN, bool F32>
__device__ __forceinline__ void stage_out_tile(const ConvKParams& p, float (&acc)[BN / 2], const float* sbias, uint8_t* stage,
                                               int row0, int c0) {
  constexpr int kEsz = F32 ? 4 : 2, kBox = y_box_bytes(BN, kEsz), kCols = kBox / kEsz;
  constexpr int kGroupBytes = (F32 ? 64 : 128) * kBox;
  // this thread's rows are 8 apart and the staging half is 1024-byte aligned, so the XOR term is the same for all of them;
  // the empty asm keeps the 16 per-column offsets below from being hoisted out of the tile loop and held in registers
  int xr = (((row0 * kBox) >> 7) & (kBox / 16 - 1)) << 4;
  asm volatile("" : "+r"(xr));
  uint8_t* base = stage + row0 * kBox;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};
    if (p.bias != nullptr) {
      const float2 b = *reinterpret_cast<const float2*>(sbias + 8 * j + c0);
      v[0] += b.x;
      v[1] += b.y;
      v[2] += b.x;
      v[3] += b.y;
    }
    activate(p, v);
    uint8_t* dst = base + (8 * j / kCols) * kGroupBytes + ((((8 * j) % kCols + c0) * kEsz) ^ xr);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (F32) *reinterpret_cast<float2*>(dst + 8 * i * kBox) = make_float2(v[2 * i], v[2 * i + 1]);
      else *reinterpret_cast<uint32_t*>(dst + 8 * i * kBox) = pack2<T>(v[2 * i], v[2 * i + 1]);
    }
  }
}

// stmatrix .trans: the four 8 x 8 b16 blocks whose mma fragments are r0..r3, each stored transposed -- lane 8 k + i gives the
// address of row i of block k, which receives column i of the fragment block (16 bytes)
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}

// TMA-store epilogue of a transposed BN = 64 halo tile (see mma_kblock_t): bias + activation on one accumulator half, which
// holds channels r0 + 8 i and pixels 8 j + c0, + 1 (j < 8) of a 64-pixel half, rounded to the output dtype and written
// pixel-major into the same boxes as stage_out_tile, from pixel row px0 of the staging half on.  bf16: the four 8 x 8
// (channel x pixel) blocks of j = 2 jj, 2 jj + 1 go out in one stmatrix .trans, each as eight 16-byte units (one pixel's 8
// channels, one swizzled unit per 128-byte row): conflict-free, where 2-byte stores would hit one bank for every pixel.
template <typename T, bool F32>
__device__ __forceinline__ void stage_out_tile_t(const ConvKParams& p, float (&acc)[32], const float* sbias, uint8_t* stage, int px0,
                                                 int r0, int c0, int lane) {
  float b[2] = {0.f, 0.f};
  if (p.bias != nullptr) {
    b[0] = sbias[r0];
    b[1] = sbias[r0 + 8];
  }
  if constexpr (F32) {
    constexpr int kBox = y_box_bytes(64, 4), kCols = kBox / 4, kGroupBytes = 64 * kBox;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v[4] = {acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]};   // (channel r0 + 8 (m / 2), pixel + m % 2)
      if (p.bias != nullptr) {
#pragma unroll
        for (int m = 0; m < 4; ++m) v[m] += b[m / 2];
      }
      activate(p, v);
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int q = px0 + 8 * j + c0 + (m & 1), n = r0 + 8 * (m >> 1);
        *reinterpret_cast<float*>(stage + (n / kCols) * kGroupBytes + q * kBox + (((n % kCols) * 4) ^ ((q & 7) << 4))) = v[m];
      }
    }
  } else {
    // lane 8 k + i: row i (pixel 8 j + i) of block k = (j = 2 jj + k / 2, channels 8 (2 w + k % 2) ..., w = r0 / 16); the box
    // rows are 128 bytes and 8-row aligned, so the swizzle XORs the 16-byte unit with i
    const int k = lane >> 3, i = lane & 7;
    const uint32_t dst = smem_u32(stage) + (uint32_t)(px0 + 8 * (k >> 1) + i) * 128u + ((uint32_t)((2 * (r0 >> 4) + (k & 1)) ^ i) << 4);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      float v[8];                                    // v[m] = channel r0 + 8 ((m / 2) % 2), pixel 8 (2 jj + m / 4) + c0 + m % 2
#pragma unroll
      for (int m = 0; m < 8; ++m) v[m] = acc[8 * jj + m];
      if (p.bias != nullptr) {
#pragma unroll
        for (int m = 0; m < 8; ++m) v[m] += b[(m >> 1) & 1];
      }
      activate(p, v);
      stmatrix_x4_trans(dst + (uint32_t)jj * 16u * 128u, pack2<T>(v[0], v[1]), pack2<T>(v[2], v[3]), pack2<T>(v[4], v[5]),
                        pack2<T>(v[6], v[7]));
    }
  }
}

// One K block of a 128-row tile: 2 x KSTEPS k16 MMAs (rows 0-63 from descriptor ad, rows 64-127 from ad + a_hi, the same
// B operand), issued back to back as ONE commit group.  KSTEPS must be known at compile time: an MMA under a runtime
// condition makes ptxas split the group and inject warpgroup.arrive around it (warning C7519).  LO: the same group with the
// rows 0-63 MMAs only, for a tile whose rows 64-127 all lie outside the output (upper_half_dead); acc[1] is left as it is.
// F16: fp16 operands.
template <int BN, int KSTEPS, bool LO = false, bool F16 = false>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][BN / 2], uint64_t ad, uint32_t a_hi, uint64_t bd, uint32_t scale_d) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    const uint32_t sd = k == 0 ? scale_d : 1u;
    Wgmma<BN, 0, 0, F16>::mma(acc[0], ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), sd);
    if constexpr (!LO) Wgmma<BN, 0, 0, F16>::mma(acc[1], ad + (uint64_t)(a_hi + 2 * k), bd + (uint64_t)(2 * k), sd);
  }
  wgmma_commit();
}

// A tile's upper half is dead when every row 64-127 of its BW x BH x BI box (pixel-major: row = bw + BW (bh + BH bi)) is
// outside the output or beyond the box, so that nothing computed for them is ever stored.  The box rows from 64 on are the
// (bi, bh, bw) at or after row 64's in lexicographic order; the rows inside the output are a product of ranges from 0, whose
// lexicographic last is (ni - 1, nh - 1, nw - 1).  For the 8 x 16 halo tiles this is t.h0 + 8 >= Ho; the empty second tile of
// a CTA pair's last unit (placed on image N) counts as dead too.  Row 64's coordinates are worked out once per kernel: with
// the divisions done per tile, the BN-64 1x1 layers of YOLOv6-S (about 12 tiles per CTA) ran about 1 % slower on an H100.
struct Row64 {
  int w, h, i;   // box coordinates of row 64; i = BI when the box has <= 64 rows
};
__device__ __forceinline__ Row64 row64_of(const ConvKParams& p) {
  const int q = 64 / p.BW;
  return Row64{64 % p.BW, q % p.BH, p.rows <= 64 ? p.BI : q / p.BH};
}
__device__ __forceinline__ bool upper_half_dead(const ConvKParams& p, const Row64& r, const TileCoord& t) {
  const int ni = min(p.N - t.i0, p.BI), nh = min(p.Ho - t.h0, p.BH), nw = min(p.Wo - t.w0, p.BW);
  if (ni <= 0 || nh <= 0 || nw <= 0) return true;
  if (ni - 1 != r.i) return ni - 1 < r.i;
  if (nh - 1 != r.h) return nh - 1 < r.h;
  return nw - 1 < r.w;
}

// The same K block of a BN = 64 halo tile computed transposed, D[64 channels x 128 pixels]: the 64-row weight tile (wd) is the
// A operand and the input box's 128 pixel rows (xd, sixteen 8-row groups) the B operand -- one m64n128k16 per k16 step, half
// the instructions of mma_kblock<64> for the same FLOPs.  acc[h] holds pixels 64 h .. 64 h + 63 (wgmma fragment columns
// 8 j + ..., j = 8 h + j' -> acc[h][4 j' + ...]).
template <int KSTEPS, bool F16 = false>
__device__ __forceinline__ void mma_kblock_t(float (&acc)[2][32], uint64_t wd, uint64_t xd, uint32_t scale_d) {
  float(&d)[64] = reinterpret_cast<float(&)[64]>(acc);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) Wgmma<128, 0, 0, F16>::mma(d, wd + (uint64_t)(2 * k), xd + (uint64_t)(2 * k), k == 0 ? scale_d : 1u);
  wgmma_commit();
}

// MODE: 0 = one TMA box per (tap, channel block); 1 / 3 = halo input tiles (stride 1 / stride-2 column-pair view), weights
//       streamed through a ring; 2 / 4 = the same with the layer's weights resident in shared memory.  BN = the wgmma N and
//       the width of the accumulator tile.  CP: CTA-pair variant (launched as clusters of two CTAs, see ConvKParams::cpair).
//       All are compile-time so that each variant carries only its own loops.  T: the operand dtype (__nv_bfloat16 or __half).
//       The body of both kernels below, force-inlined: a call would make ptxas serialize every wgmma.
template <typename T, int BN, int MODE, bool CP>
__device__ __forceinline__ void conv_igemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmY,
                                                const ConvKParams& p) {
  constexpr bool F16 = std::is_same_v<T, __half>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + (size_t)p.a_region_bytes;
  float* sC = reinterpret_cast<float*>(sB + (size_t)p.b_region_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sC) + staging_bytes(BN));
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;
  uint64_t* a_full = empty + kMaxStages;            // halo mode rings
  uint64_t* a_empty = a_full + kMaxAStages;
  uint64_t* b_full = a_empty + kMaxAStages;
  uint64_t* b_empty = b_full + kMaxBStages;
  uint64_t* mma_turn = b_empty + kMaxBStages;       // [wg]: warpgroup wg may start the MMAs of its next tile

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr bool HALO = (MODE != 0);
  constexpr bool BRES = (MODE == 2 || MODE == 4);
  constexpr bool SWAP = (HALO && BN == 64);         // the tile is computed transposed (mma_kblock_t)
  using HG = HaloGeom<(MODE >= 3)>;
  // schedule: the CTA (or CTA pair) takes units unit0, unit0 + ustep, ...; in pair mode this CTA computes M tile `rank` of a unit
  const int rank = CP ? (int)cluster_ctarank() : 0;
  const int unit0 = CP ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int ustep = CP ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  auto coord = [&](int unit) { return CP ? decode_unit(p, unit, rank) : decode_tile(p, unit); };
  // weight (B) loads: this CTA's half of the tile, multicast to both CTAs of the pair
  auto load_b = [&](uint8_t* dst, uint64_t* bar, int k, int n0, int plane) {
    if (CP) tma_load_3d_mc(dst + rank * p.b_rows * p.kb_bytes, &tmB, bar, k, n0 + rank * p.b_rows, plane, 3);
    else tma_load_3d(dst, &tmB, bar, k, n0, plane);
  };

  if (warp == 0) {
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      if (p.tma_store) tma_prefetch_desc(&tmY);
    }
    // full barriers: the producer's expect_tx arrival; empty barriers: one arrival from the warpgroup that owns the stage's
    // tile (in both CTAs when the weight stages are multicast; the input-only a_empty ring of the halo modes stays per CTA);
    // mma_turn: all 128 threads of the other consumer warpgroup
    constexpr int kRingSlots = 2 * kMaxStages + 2 * kMaxAStages + 2 * kMaxBStages;
    for (int i = lane; i < kRingSlots + 2; i += 32) {
      const bool is_b_empty = (i >= kMaxStages && i < 2 * kMaxStages) || (i >= 2 * kMaxStages + 2 * kMaxAStages + kMaxBStages && i < kRingSlots);
      mbar_init(&bars[i], i >= kRingSlots ? 128u : (is_b_empty && CP) ? 2u : 1u);
    }
    static_assert((kRingSlots + 2) * sizeof(uint64_t) <= 1024, "barriers overflow their 1 KB of shared memory");
    fence_mbar_init();
  }
  if (CP) cluster_sync_all();   // the peer's barriers are initialised before anything multicasts into it or arrives on them
  else __syncthreads();

  const int kblocks = p.npairs * p.taps * p.cin_blocks;

  if (warp < 4) {
    producer_regs();
    if (warp == 0) {
      // ================================ TMA producer ================================
      // The whole warp walks the schedule (keeps control flow convergent so addresses / coordinates
      // live in uniform registers); one elected lane arms the barrier and issues the TMA loads.
      // It fills the rings in tile order; which consumer warpgroup owns a tile does not concern it.
      if constexpr (HALO) {
        int sa = 0, sb = 0;
        uint32_t pha = 0, phb = 0;
        bool first = true;
        const uint32_t a_tx = (uint32_t)HG::kBytes, b_tx = (uint32_t)(BN * 128);
        for (int tile = unit0; tile < p.num_tiles; tile += ustep) {
          const TileCoord t = coord(tile);
          int slot = 0;
          for (int pi = 0; pi < p.npairs; ++pi) {
            const int pa = kPairA[6 - p.npairs + pi], pb = kPairB[6 - p.npairs + pi];
            for (int cb = 0; cb < p.cin_blocks; ++cb) {
              mbar_wait(&a_empty[sa], pha ^ 1);
              if (elect_one()) {
                mbar_expect_tx(&a_full[sa], a_tx);
                tma_load_5d(sA + (size_t)sa * HG::kStageBytes, &tmA, &a_full[sa], cb * 64, t.w0 - 1, t.h0 * HG::SH - 1, t.i0, pa);
              }
              __syncwarp();
              if (++sa == p.a_stages) { sa = 0; pha ^= 1; }
              for (int tap = 0; tap < HG::TAPS; ++tap) {
                if (HG::SH == 2 && (tap % HG::KW) == 0 && cb < p.skip_cb) continue;     // all-zero weight block
                if constexpr (BRES) {
                  if (first && elect_one()) {
                    mbar_expect_tx(&b_full[slot], b_tx);
                    load_b(sB + (size_t)slot * p.b_stage_bytes, &b_full[slot], tap * p.Cin + cb * 64, t.n0, pb);
                  }
                  __syncwarp();
                } else {
                  mbar_wait(&b_empty[sb], phb ^ 1);
                  if (elect_one()) {
                    mbar_expect_tx(&b_full[sb], b_tx);
                    load_b(sB + (size_t)sb * p.b_stage_bytes, &b_full[sb], tap * p.Cin + cb * 64, t.n0, pb);
                  }
                  __syncwarp();
                  if (++sb == p.b_stages) { sb = 0; phb ^= 1; }
                }
                ++slot;
              }
            }
          }
          first = false;
        }
      } else {
        int stage = 0;
        uint32_t phase = 0;
        const uint32_t tx = (uint32_t)(p.rows * p.kb_bytes + BN * p.kb_bytes);
        for (int tile = unit0; tile < p.num_tiles; tile += ustep) {
          const TileCoord t = coord(tile);
          for (int pi = 0; pi < p.npairs; ++pi) {
            const int pa = kPairA[6 - p.npairs + pi], pb = kPairB[6 - p.npairs + pi];
            for (int tap = 0; tap < p.taps; ++tap) {
              const int r = tap / p.kw, s = tap - r * p.kw;
              const int cx = t.w0 * p.stride_w + s - p.pad_w;
              const int cy = t.h0 * p.stride + r - p.pad;
              for (int cb = 0; cb < p.cin_blocks; ++cb) {
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {
                  mbar_expect_tx(&full[stage], tx);
                  tma_load_5d(sA + (size_t)stage * p.a_stage_bytes, &tmA, &full[stage], cb * p.kb_elems, cx, cy, t.i0, pa);
                  load_b(sB + (size_t)stage * p.b_stage_bytes, &full[stage], tap * p.Cin + cb * p.kb_elems, t.n0, pb);
                }
                __syncwarp();
                if (++stage == p.stages) {
                  stage = 0;
                  phase ^= 1;
                }
              }
            }
          }
        }
      }
    }
  } else {
    consumer_regs();
    // ================================ consumers ================================
    // Ping-pong: the CTA's local tile j (its j-th schedule unit) belongs to warpgroup j & 1, which computes all 128 rows of
    // it.  The two take turns on the tensor cores: a warpgroup issues the first MMA of a tile only once the other has
    // committed the last MMA of the preceding tile (mma_turn), so each tile's epilogue runs under the next tile's MMAs.
    // Within a tile one wgmma group is kept in flight: after committing K block i the warpgroup waits for block i - 1 and
    // only then releases that block's shared memory.  Only the last group of a tile is waited for in full, before the
    // epilogue.  A warpgroup steps over the ring stages of the other's tiles (a tile takes the same number of stages
    // throughout a launch) and never waits on their barriers.
    const int wg = (warp >> 2) - 1;
    const int ct = (int)threadIdx.x - 128 * (wg + 1);   // 0 .. 127
    const bool arrive_lane = ct == 0;                    // one arrival per tile owner on the empty barriers
    // a weight-carrying stage is released in both CTAs of a pair (the peer's producer multicasts into this CTA's copy)
    auto release_b = [&](uint64_t* bar) {
      mbar_arrive(bar);
      if (CP) mbar_arrive_cluster(bar, (uint32_t)(rank ^ 1));
    };
    auto skip_stages = [](int& s, uint32_t& ph, int n, int ring) {
      s += n;
      ph ^= (uint32_t)(s / ring) & 1u;
      s %= ring;
    };
    float acc[2][BN / 2];                                // rows 0-63 and 64-127 of the tile
    const uint32_t a_base = smem_u32(sA) >> 4, b_base = smem_u32(sB) >> 4;
    const int num_tiles = p.num_tiles, ksteps = p.ksteps, nstages = p.stages;
    // ring stages of one tile: mode 0: kblocks; halo modes: pcs input stages and b_tile weight stages (streamed weights)
    const int pcs = p.npairs * p.cin_blocks;
    const int b_tile = p.npairs * (p.cin_blocks * HG::TAPS - (HG::SH == 2 ? (HG::TAPS / HG::KW) * p.skip_cb : 0));
    int stage = 0;
    uint32_t phase = 0;
    int sa = 0, sb = 0;
    uint32_t pha = 0, phb = 0, turn_ph = 0;
    bool first = true;
    float* sCw = sC + wg * 64 * stage_pitch(BN);         // this warpgroup's half of the staging tile
    float* sbias = sCw + 64 * BN;                        // TMA-store epilogue: the tile's bias, after the staged tile
    const Row64 row64 = row64_of(p);
    for (int tile = unit0 + wg * ustep; tile < num_tiles; tile += 2 * ustep) {
      const TileCoord t = coord(tile);
      // TMA-store epilogue: the tile's bias goes to shared memory before the MMAs (this warpgroup's last epilogue read its
      // previous contents before its final barrier), so that its load latency hides under the wait for the tensor cores
      if (p.tma_store && p.bias != nullptr && ct < BN) sbias[ct] = __ldg(p.bias + t.n0 + ct);
      // rows 64-127 lie wholly outside the output (the last tile row of a map with Ho % 16 in 1..8, a box of <= 64 rows): the
      // K loop issues only the rows 0-63 MMAs and the epilogue skips acc[1].  The transposed BN = 64 halo tiles keep one
      // m64n128 per k16 step over all 128 pixels.
      const bool dead_hi = !SWAP && upper_half_dead(p, row64, t);
      if (tile != unit0) {                               // the other warpgroup owns the preceding tile
        if constexpr (HALO) {
          skip_stages(sa, pha, pcs, p.a_stages);
          if (!BRES) skip_stages(sb, phb, b_tile, p.b_stages);
        } else {
          skip_stages(stage, phase, kblocks, nstages);
        }
        mbar_wait(&mma_turn[wg], turn_ph);
        turn_ph ^= 1;
      }
      // The tile's K loop, in two copies whose commit groups hold a fixed number of MMAs each (see mma_kblock): lo_only =
      // std::true_type issues rows 0-63 only.  The K order, stage releases and hand-over are the same in both.
      auto mainloop = [&](auto lo_only) {
        [[maybe_unused]] constexpr bool LO = decltype(lo_only)::value;   // (the transposed BN = 64 tiles ignore it)
        if constexpr (HALO) {
          // A descriptors walk the halo tile: 8-row groups are the 8 pixels of one output row, SH halo rows apart;
          // tap (r,s) shifts the start address by (W r + s) pixels, rows 64-127 start 8 output rows further.  At BN = 64 the same
          // descriptor is the B operand and spans all 16 groups.
          const uint32_t row_bytes = (uint32_t)(HG::W * 128 * HG::SH);
          const uint64_t desc_a = wgmma_desc(16u, row_bytes, 1u);
          const uint64_t desc_b = wgmma_desc(16u, 1024u, 1u);
          const uint32_t halo_step = (uint32_t)HG::kStageBytes >> 4, b_step = (uint32_t)p.b_stage_bytes >> 4;
          [[maybe_unused]] const uint32_t a_hi = 8u * (row_bytes >> 4);
          const int skip_cb = p.skip_cb, cin_blocks = p.cin_blocks, b_stages = p.b_stages;
          int slot = 0;
          uint32_t started = 0;
          // Stages whose MMAs may still be in flight: the B stage of the last committed group and the A stage of the previous
          // channel block.  Each is released once a later group has been committed and wgmma_wait<1> has returned, so the
          // pipe never drains at a channel-block boundary; the one full wait per tile comes before the epilogue.
          int prev_sb = -1, prev_sa = -1;
          for (int pc = 0; pc < pcs; ++pc) {
            mbar_wait(&a_full[sa], pha);
            const uint32_t a0 = a_base + (uint32_t)sa * halo_step;
            const bool skip_s0 = (HG::SH == 2) && (pc % cin_blocks) < skip_cb;      // this channel block of the s = 0 taps is all zero
#pragma unroll
            for (int tap = 0; tap < HG::TAPS; ++tap) {
              if (HG::SH == 2 && (tap % HG::KW) == 0 && skip_s0) continue;
              const int bs = BRES ? slot : sb;
              // resident weights were loaded during the CTA's first tile; each warpgroup waits for them before its first tile
              if (!BRES || first) mbar_wait(&b_full[bs], BRES ? 0u : phb);
              const uint64_t ad = desc_a | (uint64_t)(a0 + (uint32_t)((tap / HG::KW) * HG::W + (tap % HG::KW)) * 8u);
              const uint64_t bd = desc_b | (uint64_t)(b_base + (uint32_t)bs * b_step);
              if constexpr (SWAP) mma_kblock_t<4, F16>(acc, bd, ad, started);
              else mma_kblock<BN, 4, LO, F16>(acc, ad, a_hi, bd, started);
              started = 1u;
              if (!BRES || prev_sa >= 0) {
                wgmma_wait<1>();
                if (arrive_lane) {
                  if (!BRES && prev_sb >= 0) release_b(&b_empty[prev_sb]);
                  if (prev_sa >= 0) mbar_arrive(&a_empty[prev_sa]);
                }
                prev_sa = -1;
              }
              if (!BRES) {
                prev_sb = sb;
                if (++sb == b_stages) { sb = 0; phb ^= 1; }
              }
              ++slot;
            }
            prev_sa = sa;
            if (++sa == p.a_stages) { sa = 0; pha ^= 1; }
          }
          mbar_arrive(&mma_turn[wg ^ 1]);                  // the other warpgroup may start its tile's MMAs
          wgmma_wait<0>();
          if (arrive_lane) {
            if (!BRES && prev_sb >= 0) release_b(&b_empty[prev_sb]);
            if (prev_sa >= 0) mbar_arrive(&a_empty[prev_sa]);
          }
        } else {
          const uint64_t desc = wgmma_desc(16u, (uint32_t)p.sbo_bytes, (uint32_t)p.layout_type);
          const uint32_t a_step = (uint32_t)p.a_stage_bytes >> 4, b_step = (uint32_t)p.b_stage_bytes >> 4;
          const uint32_t a_hi = (uint32_t)(64 * p.kb_bytes) >> 4;
          int prev = -1;
          for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint64_t ad = desc | (uint64_t)(a_base + (uint32_t)stage * a_step);
            const uint64_t bd = desc | (uint64_t)(b_base + (uint32_t)stage * b_step);
            const uint32_t scale_d = (uint32_t)(kb != 0);
            switch (ksteps) {          // 16-, 32- or 64-channel K blocks
              case 1: mma_kblock<BN, 1, LO, F16>(acc, ad, a_hi, bd, scale_d); break;
              case 2: mma_kblock<BN, 2, LO, F16>(acc, ad, a_hi, bd, scale_d); break;
              default: mma_kblock<BN, 4, LO, F16>(acc, ad, a_hi, bd, scale_d); break;
            }
            wgmma_wait<1>();
            if (prev >= 0 && arrive_lane) release_b(&empty[prev]);
            prev = stage;
            if (++stage == nstages) {
              stage = 0;
              phase ^= 1;
            }
          }
          mbar_arrive(&mma_turn[wg ^ 1]);                  // the other warpgroup may start its tile's MMAs
          wgmma_wait<0>();
          if (prev >= 0 && arrive_lane) release_b(&empty[prev]);
        }
      };
      if (dead_hi) mainloop(std::true_type());
      else mainloop(std::false_type());
      wgmma_fence_operand(acc[0]);
      wgmma_fence_operand(acc[1]);
      first = false;

      const int r0 = (warp & 3) * 16 + (lane >> 2);      // this thread's fragment rows r0 + 8 i (+ 64 for acc[1]) and
      const int c0 = 2 * (lane & 3);                     // columns 8 j + c0, + 1
      if (p.tma_store) {
        // ---- epilogue through the output tensor map: bias, activation and rounding in registers, the tile staged in the
        //      output dtype (bf16: all 128 rows in one pass; fp32: one 64-row pass per accumulator half), one bulk tensor
        //      store per column group.  The stores clip at the output's edges, so a dead upper half (dead_hi) is neither
        //      computed nor staged: bf16 stores whatever its staging rows hold, which lie outside the output; fp32 skips
        //      its second pass. ----
        const bool f32 = p.y_dtype == YV6_DT_F32;
        uint8_t* stage = reinterpret_cast<uint8_t*>(sCw);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (h == 1 && (!f32 || dead_hi)) break;
          if (ct == 0) bulk_wait_read();               // the last store has read the staging half
          warpgroup_bar_sync(wg);
          if constexpr (SWAP) {
            if (f32) {
              stage_out_tile_t<T, true>(p, acc[h], sbias, stage, 0, r0, c0, lane);
            } else {
              stage_out_tile_t<T, false>(p, acc[0], sbias, stage, 0, r0, c0, lane);
              stage_out_tile_t<T, false>(p, acc[1], sbias, stage, 64, r0, c0, lane);
            }
          } else if (f32) {
            stage_out_tile<T, BN, true>(p, acc[h], sbias, stage, r0, c0);
          } else {
            stage_out_tile<T, BN, false>(p, acc[0], sbias, stage, r0, c0);
            if (!dead_hi) stage_out_tile<T, BN, false>(p, acc[1], sbias, stage, r0 + 64, c0);
          }
          fence_proxy_async();
          warpgroup_bar_sync(wg);
          if (ct == 0) {
            const int gcols = y_box_bytes(BN, f32 ? 4 : 2) / (f32 ? 4 : 2);
            const int group_bytes = (f32 ? 64 : 128) * y_box_bytes(BN, f32 ? 4 : 2);
            for (int g = 0; g * gcols < BN; ++g)
              tma_store_4d(&tmY, stage + g * group_bytes, t.n0 + g * gcols, t.w0, t.h0 + h * (p.BH / 2), t.i0);
            bulk_commit();
            if (tile + 2 * ustep >= num_tiles) bulk_wait_read();   // the CTA's shared memory outlives the last store's reads
          }
        }
        continue;
      }
      // ---- chunk epilogue (residual, bf16x3 planes, outputs a tensor map cannot describe), in two 64-row passes:
      //      fragment -> this warpgroup's staging half -> coalesced 16-channel chunks with the fused tail ----
      constexpr int kChunks = BN / 16;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rows = min(64, p.rows - 64 * h);
        if (rows <= 0 || (h == 1 && dead_hi)) break;
        warpgroup_bar_sync(wg);                  // the previous pass's chunks have all been read from the staging half
        if constexpr (SWAP) {                    // transposed: channels r0 + 8 i of pixels 8 j + c0 + c
#pragma unroll
          for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int m = 0; m < 4; ++m)
              sCw[(8 * j + c0 + (m & 1)) * stage_pitch(BN) + r0 + 8 * (m >> 1)] = acc[h][4 * j + m];
          }
        } else {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              *reinterpret_cast<float2*>(sCw + (r0 + 8 * i) * stage_pitch(BN) + 8 * j + c0) =
                  make_float2(acc[h][4 * j + 2 * i], acc[h][4 * j + 2 * i + 1]);
            }
          }
        }
        warpgroup_bar_sync(wg);
        for (int item = ct; item < rows * kChunks; item += 128) {
          const int lr = item / kChunks, ch = item - lr * kChunks;
          const int row = 64 * h + lr;
          const int n = t.n0 + 16 * ch;
          const int ncol = min(16, p.Cout - n);
          if (ncol <= 0) continue;
          const int bw = row % p.BW, tq = row / p.BW;
          const int bh = tq % p.BH, bi = tq / p.BH;
          const int img = t.i0 + bi, ho = t.h0 + bh, wo = t.w0 + bw;
          if (img >= p.N || ho >= p.Ho || wo >= p.Wo) continue;
          const int64_t off = (int64_t)img * p.y_img_stride + (int64_t)ho * p.y_h_stride + (int64_t)wo * p.y_w_stride;
          const int64_t roff = (int64_t)img * p.res_img_stride + (int64_t)ho * p.res_h_stride + (int64_t)wo * p.res_w_stride;
          const float4* src = reinterpret_cast<const float4*>(sCw + lr * stage_pitch(BN) + 16 * ch);
          uint32_t r[16];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 f = src[q];
            r[4 * q + 0] = __float_as_uint(f.x);
            r[4 * q + 1] = __float_as_uint(f.y);
            r[4 * q + 2] = __float_as_uint(f.z);
            r[4 * q + 3] = __float_as_uint(f.w);
          }
          float v[16];
          epilogue_math<T>(p, r, n, ncol, roff, v);
          store_chunk<T>(p, off, n, ncol, v);
        }
      }
    }
  }
  // neither CTA of a pair may exit while its peer can still multicast into it or arrive on its barriers
  if (CP) cluster_sync_all();
}

template <int BN, int MODE, bool CP>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmY, const ConvKParams p) {
  conv_igemm_body<__nv_bfloat16, BN, MODE, CP>(tmA, tmB, tmY, p);
}

// fp16 operands (yv6_conv_desc.reserved0 = YV6_DT_F16): fp16 wgmma, fp16 input / residual / output, fp32 accumulation
template <int BN, int MODE, bool CP>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_f16_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmY, const ConvKParams p) {
  conv_igemm_body<__half, BN, MODE, CP>(tmA, tmB, tmY, p);
}

// ------------------------------------------------------------------------------------------------
// host side: tile planning, tensor-map encoding, launch
// ------------------------------------------------------------------------------------------------
struct ConvPlan {
  ConvKParams k;
  int grid;
  size_t smem_bytes;
  CUtensorMapSwizzle swz;
  bool f16;               // fp16 operands (conv_f16_igemm_kernel); the tile plan is the same as for bf16
};

// wgmma N of the kernel variants (accumulator registers per consumer thread = BN: two m64 halves of BN / 2)
constexpr int kBNs[4] = {32, 64, 96, 128};

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

static int plan_conv(const yv6_handle* h, const yv6_conv_desc* d, ConvPlan* plan) {
  YV6_REQUIRE(d != nullptr, "conv: null descriptor");
  YV6_REQUIRE(d->x && d->w && d->y, "conv: null tensor pointer");
  YV6_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0, "conv: bad input shape %dx%dx%d", d->N, d->H, d->W);
  YV6_REQUIRE(d->Cin > 0 && d->Cin % 16 == 0, "conv: Cin=%d must be a positive multiple of 16", d->Cin);
  YV6_REQUIRE(d->x_c_total >= d->Cin && d->x_c_total % 8 == 0, "conv: bad x_c_total=%d", d->x_c_total);
  YV6_REQUIRE(d->Cout > 0, "conv: Cout=%d", d->Cout);
  YV6_REQUIRE(d->kh >= 1 && d->kh <= 3 && d->kw >= 1 && d->kw <= 3, "conv: kernel %dx%d unsupported", d->kh, d->kw);
  YV6_REQUIRE(d->stride == 1 || d->stride == 2, "conv: stride %d unsupported", d->stride);
  YV6_REQUIRE(d->stride_w >= 0 && d->stride_w <= 2, "conv: stride_w %d unsupported", d->stride_w);
  const int stride_w = d->stride_w > 0 ? d->stride_w : d->stride;
  YV6_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "conv: nsplit must be 1 or 3");
  YV6_REQUIRE((reinterpret_cast<uintptr_t>(d->x) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->w) & 15) == 0,
              "conv: x / w must be 16-byte aligned");
  // reserved0 = operand dtype: 0 (bf16) or YV6_DT_F16 (one plane)
  YV6_REQUIRE(d->reserved0 == 0 || d->reserved0 == YV6_DT_F16, "conv: operand dtype %d must be 0 (bf16) or YV6_DT_F16", d->reserved0);
  plan->f16 = d->reserved0 == YV6_DT_F16;
  YV6_REQUIRE(!plan->f16 || d->nsplit == 1, "conv: fp16 operands need nsplit == 1");
  YV6_REQUIRE(d->y_dtype == (plan->f16 ? YV6_DT_F16 : YV6_DT_BF16) || d->y_dtype == YV6_DT_F32, "conv: bad y_dtype %d", d->y_dtype);

  ConvKParams& k = plan->k;
  memset(&k, 0, sizeof(k));
  k.N = d->N;
  // pad_w < 0 means "same as pad" (square padding); out_h/out_w > 0 override the conv arithmetic (used by
  // the parity sub-problems of a stride-2 dgrad, whose far-side reads rely on TMA zero fill)
  const int pad_w = (d->pad_w == YV6_PAD_SAME) ? d->pad : d->pad_w;
  k.Ho = d->out_h > 0 ? d->out_h : (d->H + 2 * d->pad - d->kh) / d->stride + 1;
  k.Wo = d->out_w > 0 ? d->out_w : (d->W + 2 * pad_w - d->kw) / stride_w + 1;
  YV6_REQUIRE(k.Ho > 0 && k.Wo > 0, "conv: empty output");
  k.Cout = d->Cout;
  k.Cin = d->Cin;
  k.taps = d->kh * d->kw;
  k.kw = d->kw;
  k.stride = d->stride;
  k.stride_w = stride_w;
  k.pad = d->pad;
  k.pad_w = pad_w;

  // K block = largest of 64/32/16 channels dividing Cin -> 128/64/32-byte swizzle
  k.kb_elems = (d->Cin % 64 == 0) ? 64 : (d->Cin % 32 == 0) ? 32 : 16;
  k.kb_bytes = k.kb_elems * 2;
  k.ksteps = k.kb_elems / 16;
  k.cin_blocks = d->Cin / k.kb_elems;
  k.sbo_bytes = 8 * k.kb_bytes;
  k.layout_type = (int)wgmma_layout(k.kb_bytes);
  plan->swz = (k.kb_bytes == 128) ? CU_TENSOR_MAP_SWIZZLE_128B
              : (k.kb_bytes == 64) ? CU_TENSOR_MAP_SWIZZLE_64B
                                   : CU_TENSOR_MAP_SWIZZLE_32B;
  k.npairs = (d->nsplit == 3) ? 6 : 1;

  // M tiling: BW x BH x BI box of output pixels, <= 128 rows, fewest tiles wins
  if (d->force_bw > 0) {
    k.BW = d->force_bw;
    k.BH = std::max(1, d->force_bh);
    k.BI = std::max(1, d->force_bi);
    YV6_REQUIRE(k.BW * k.BH * k.BI <= kTileRows && k.BW * stride_w <= 256 && k.BH * d->stride <= 256,
                "conv: forced tile %dx%dx%d invalid", k.BW, k.BH, k.BI);
  } else {
    long best_tiles = -1, best_box_tiles = -1;
    int bestw = 1, besth = 1, besti = 1, boxw = 0, boxh = 0;
    const int maxbw = std::min(std::min(k.Wo, kTileRows), 256 / stride_w);
    for (int bw = 1; bw <= maxbw; ++bw) {
      const int maxbh = std::min(std::min(k.Ho, kTileRows / bw), 256 / d->stride);
      for (int bh = 1; bh <= maxbh; ++bh) {
        int bi = 1;
        if (bw >= k.Wo && bh >= k.Ho) bi = std::max(1, std::min(d->N, kTileRows / (bw * bh)));
        long tiles = (long)ceil_div(k.Wo, bw) * ceil_div(k.Ho, bh) * ceil_div(d->N, bi);
        if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && bw > bestw)) {
          best_tiles = tiles;
          bestw = bw;
          besth = bh;
          besti = bi;
        }
      }
    }
    // "box" tiles: 128 rows of power-of-two width, whose 16-row wgmma fragments are boxes of the output; preferred
    // within 8 % of the best
    for (int bw = 1; bw <= std::min(kTileRows, 256 / stride_w); bw <<= 1) {
      const int bh = kTileRows / bw;
      if (bh * d->stride > 256) continue;
      long tiles = (long)ceil_div(k.Wo, bw) * ceil_div(k.Ho, bh) * d->N;
      if (best_box_tiles < 0 || tiles < best_box_tiles || (tiles == best_box_tiles && bw > boxw)) {
        best_box_tiles = tiles;
        boxw = bw;
        boxh = bh;
      }
    }
    if (best_box_tiles > 0 && best_box_tiles * 100 <= best_tiles * 108 && d->force_bi == 0) {
      bestw = boxw;
      besth = boxh;
      besti = 1;
    }
    k.BW = bestw;
    k.BH = besth;
    k.BI = besti;
  }
  // halo mode: 3x3 stride-1 with 64-channel K blocks and an 8x16 output tile; taken when its fixed tile
  // shape costs at most 25% more tiles than the best free-form box (it moves ~6x fewer A bytes)
  k.halo = 0;
  if (d->kh == 3 && d->kw == 3 && d->stride == 1 && stride_w == 1 && d->pad == 1 && pad_w == 1 && d->out_h == 0 && d->out_w == 0 &&
      d->Cin % 64 == 0 && d->force_bw == 0 && d->force_halo >= 0) {
    const long generic = (long)ceil_div(k.Wo, k.BW) * ceil_div(k.Ho, k.BH) * ceil_div(d->N, k.BI);
    const long halo_tiles = (long)ceil_div(k.Wo, 8) * ceil_div(k.Ho, 16) * d->N;
    if (d->force_halo > 0 || halo_tiles * 4 <= generic * 5) {
      k.halo = 1;
      k.BW = 8;
      k.BH = 16;
      k.BI = 1;
    }
  }
  // halo 2: the column-pair view of a 3x3 stride-2 conv (3x2 kernel, stride (2, 1), pad (1, 1), out_w = W), same 8 x 16 tile
  // over a 9 x 33 box: ~2.6x fewer A bytes from L2 than one box per tap.  pair_view additionally promises that the weights of
  // the left tap are zero over the even pixel's channels [0, Cin/2): whole 64-channel blocks of zeros are skipped.
  k.skip_cb = 0;
  if (d->kh == 3 && d->kw == 2 && d->stride == 2 && stride_w == 1 && d->pad == 1 && pad_w == 1 && d->out_w == d->W && d->out_h == 0 &&
      d->Cin % 64 == 0 && d->force_bw == 0 && d->force_halo >= 0 && d->H % 2 == 0) {
    const long generic = (long)ceil_div(k.Wo, k.BW) * ceil_div(k.Ho, k.BH) * ceil_div(d->N, k.BI);
    const long halo_tiles = (long)ceil_div(k.Wo, 8) * ceil_div(k.Ho, 16) * d->N;
    // auto: up to 128 real input channels and where the fixed tile wastes < 25 %; beyond that the
    // weight operand dominates the L2 -> shared-memory traffic and the plain stride-2 mainloop (fewer, wider K blocks) wins
    if (d->force_halo > 0 || (halo_tiles * 4 <= generic * 5 && d->Cin <= 256)) {
      k.halo = 2;
      k.BW = 8;
      k.BH = 16;
      k.BI = 1;
      if (d->pair_view && (d->Cin / 2) % 64 == 0) k.skip_cb = d->Cin / 128;
    }
  }
  const long m_tiles = (long)ceil_div(k.Wo, k.BW) * ceil_div(k.Ho, k.BH) * ceil_div(d->N, k.BI);
  // N tiling: BN one of the kernel variants' widths; pick the one whose wave count x tile cost is smallest
  // (a 448-tile layer on 132 SMs runs 4 waves at BN=128 but 7 half-cost waves at BN=64).
  if (d->force_bn > 0) {
    YV6_REQUIRE(d->force_bn == 32 || d->force_bn == 64 || d->force_bn == 96 || d->force_bn == 128, "conv: force_bn must be 32, 64, 96 or 128");
    k.BN = d->force_bn;
  } else {
    double best_cost = -1;
    int best_bn = 0;
    for (int i = 3; i >= 0; --i) {
      const int bn = kBNs[i];
      if (bn < 64 && d->Cout > bn) continue;       // N splits narrower than 64 re-read the A tile for too little work
      const long tiles = m_tiles * ceil_div(d->Cout, bn);
      const double waves = (double)ceil_div((int)std::min<long>(tiles, 1l << 30), h->num_sms);
      const double cost = waves * (bn + 48.0);  // +48: per-tile fixed cost and A re-reads favour wide tiles
      if (best_cost < 0 || cost < best_cost - 1e-9) {
        best_cost = cost;
        best_bn = bn;
      }
    }
    k.BN = best_bn;
  }
  YV6_REQUIRE(k.BN >= 16, "conv: could not choose BN for Cout=%d", d->Cout);
  k.tiles_n = ceil_div(d->Cout, k.BN);
  k.rows = k.BW * k.BH * k.BI;
  k.tiles_w = ceil_div(k.Wo, k.BW);
  k.tiles_h = ceil_div(k.Ho, k.BH);
  k.tiles_i = ceil_div(d->N, k.BI);
  YV6_REQUIRE(m_tiles * k.tiles_n < (1l << 30), "conv: too many tiles");
  k.m_tiles = (int)m_tiles;
  // CTA pairs (force_pair = 1: on whenever there are two M tiles): the weight tile is loaded once per pair and multicast, which
  // halves the L2 -> shared-memory weight traffic.  Auto mode does not take them: on the H100 the YOLOv6-S bs32 step with pairs
  // on the weight-heavy layers (3x3 stride 1 over >= 128 channels, stride-2 halo from 128 output channels) ran at 4.3 k images/s
  // against 5.3 k without (the pair's CTAs advance in lockstep and the cluster grid leaves SMs idle on the partial last wave).
  k.cpair = (m_tiles >= 2 && h->max_clusters > 0 && d->force_pair > 0) ? 1 : 0;
  k.b_rows = k.cpair ? k.BN / 2 : k.BN;
  // schedule units: tiles, or (two consecutive M tiles) x N tile for CTA pairs
  k.num_tiles = k.cpair ? (int)(((m_tiles + 1) / 2) * k.tiles_n) : (int)(m_tiles * k.tiles_n);

  // smem ring(s)
  k.a_stage_bytes = kTileRows * k.kb_bytes;
  k.b_stage_bytes = ((k.BN * k.kb_bytes + 1023) / 1024) * 1024;
  const int budget = h->max_smem_optin - 1024 - 1024 - staging_bytes(k.BN);
  if (k.halo) {
    const int halo_stage = (k.halo == 2) ? HaloGeom<true>::kStageBytes : HaloGeom<false>::kStageBytes;
    const int min_a = (k.halo == 2) ? 2 : 3;          // A stages that must fit next to resident weights
    // B tiles one output tile consumes (halo 2: six taps, minus the all-zero blocks of the three left taps)
    const int b_tiles = (k.halo == 2) ? k.npairs * (k.cin_blocks * 6 - 3 * k.skip_cb) : k.npairs * k.cin_blocks * 9;
    k.b_resident = (k.tiles_n == 1 && b_tiles <= kMaxBStages && d->force_stages == 0 &&
                    (long)b_tiles * k.b_stage_bytes + min_a * halo_stage <= budget) ? 1 : 0;
    if (k.b_resident) {
      k.b_stages = b_tiles;
      k.a_stages = std::min(kMaxAStages, (budget - b_tiles * k.b_stage_bytes) / halo_stage);
    } else {
      k.a_stages = (k.halo == 1 && budget - 3 * halo_stage >= 3 * k.b_stage_bytes) ? 3 : 2;
      k.b_stages = std::min(kMaxBStages, (budget - k.a_stages * halo_stage) / k.b_stage_bytes);
      if (d->force_stages > 0) k.b_stages = std::min(k.b_stages, std::max(2, d->force_stages));
    }
    YV6_REQUIRE(k.a_stages >= 2 && k.b_stages >= 2, "conv(halo): not enough shared memory");
    k.stages = k.b_stages;
    k.a_region_bytes = k.a_stages * halo_stage;
    k.b_region_bytes = k.b_stages * k.b_stage_bytes;
  } else {
    const int stage_bytes = k.a_stage_bytes + k.b_stage_bytes;
    int stages = std::min(kMaxStages, budget / stage_bytes);
    if (d->force_stages > 0) stages = std::min(stages, d->force_stages);
    YV6_REQUIRE(stages >= 2, "conv: not enough shared memory for a 2-stage pipeline");
    k.stages = stages;
    k.a_region_bytes = stages * k.a_stage_bytes;
    k.b_region_bytes = stages * k.b_stage_bytes;
  }
  plan->smem_bytes = (size_t)k.a_region_bytes + k.b_region_bytes + staging_bytes(k.BN) + 1024 + 1024;

  k.act = d->act;
  k.y_dtype = d->y_dtype;
  k.fast_act = (d->y_dtype == YV6_DT_BF16 && d->nsplit != 3) ? 1 : 0;   // (not for fp16: 2^-11 is half its ulp)
  k.out_planes = (d->nsplit == 3 && d->y_dtype == YV6_DT_BF16) ? 3 : 1;
  k.res_planes = (d->nsplit == 3) ? 3 : 1;
  k.y = d->y;
  k.y_img_stride = d->y_img_stride;
  k.y_h_stride = d->y_h_stride;
  k.y_w_stride = d->y_w_stride;
  k.y_plane_stride = d->y_plane_stride;
  k.res = d->res;
  k.alpha = d->alpha;
  k.res_img_stride = d->res_img_stride;
  k.res_h_stride = d->res_h_stride;
  k.res_w_stride = d->res_w_stride;
  k.res_plane_stride = d->res_plane_stride;
  k.bias = d->bias;

  // Output through a tensor map (C, W, H, N) with boxes of (box_bytes / element size) channels x the BW x BH x BI tile:
  // needs one output plane, no residual, a 16-byte aligned base and strides, a pixel's Cout outputs ending on a 16-byte
  // boundary, and in fp32 (where one staging half holds 64 rows) a 128-row tile split into two 64-row boxes along H.
  // Measured on an H100 SXM, tests/test_gpu_forward_launches.py: with the map's dims[0] = Cout = 12, the bf16 1x1 conv
  // backbone.lite_effiblock_2.0.conv_pw_2 of YOLOv6Lite-S (2 x 128 x 128, output [2, 32, 32, 16], slice [0, 12)) also
  // stored channels 12..15 (zeros) of all 8192 of its pixels x 4, and the same conv of YOLOv6Lite-L at 192 x 320 all
  // 122880: the store did not clip at the end of the 24-byte channel row.  Those outputs take the chunk epilogue.
  {
    const int esz = d->y_dtype == YV6_DT_F32 ? 4 : 2;
    const int64_t strides[3] = {d->y_w_stride * esz, d->y_h_stride * esz, d->y_img_stride * esz};
    bool ok = k.out_planes == 1 && d->res == nullptr && (reinterpret_cast<uintptr_t>(d->y) & 15) == 0 && (d->Cout * esz) % 16 == 0;
    for (int64_t s : strides) ok = ok && s > 0 && s % 16 == 0 && s < (1ll << 40);
    if (esz == 4) ok = ok && k.BI == 1 && k.BH % 2 == 0 && k.BW * k.BH == kTileRows;
    k.tma_store = ok ? 1 : 0;
  }

  if (k.cpair) {   // grid counts CTAs: two per unit
    int clusters = std::min(k.num_tiles, h->max_clusters);
    if (d->force_grid > 0) clusters = std::min(k.num_tiles, std::max(1, d->force_grid / 2));
    plan->grid = 2 * clusters;
  } else {
    plan->grid = std::min(k.num_tiles, h->num_sms);
    if (d->force_grid > 0) plan->grid = std::min(k.num_tiles, d->force_grid);
  }
  return YV6_OK;
}

}  // namespace yv6

using namespace yv6;

using ConvKernelFn = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const ConvKParams);
#define YV6_CONV_MODES(K, BN, CP) {K<BN, 0, CP>, K<BN, 1, CP>, K<BN, 2, CP>, K<BN, 3, CP>, K<BN, 4, CP>}
#define YV6_CONV_TABLE(K)                                                                                              \
  {{YV6_CONV_MODES(K, 32, false), YV6_CONV_MODES(K, 64, false), YV6_CONV_MODES(K, 96, false), YV6_CONV_MODES(K, 128, false)}, \
   {YV6_CONV_MODES(K, 32, true), YV6_CONV_MODES(K, 64, true), YV6_CONV_MODES(K, 96, true), YV6_CONV_MODES(K, 128, true)}}
// [fp16 operands][CTA pair][BN index: 32, 64, 96, 128][mode]
static const ConvKernelFn kConvKernels[2][2][4][5] = {YV6_CONV_TABLE(conv_igemm_kernel), YV6_CONV_TABLE(conv_f16_igemm_kernel)};
#undef YV6_CONV_TABLE
#undef YV6_CONV_MODES

// Once per device: opt the kernels in to the large dynamic shared memory and ask how many 2-CTA clusters of the conv kernel
// (one CTA per SM) can be co-resident -- the grid of the pair variants.
static int conv_configure(yv6_handle* h) {
  if (h->configured & YV6_CFG_CONV) return YV6_OK;
  for (const auto& by_pair : kConvKernels)
    for (const auto& by_bn : by_pair)
      for (const auto& by_mode : by_bn)
        for (ConvKernelFn fn : by_mode)
          YV6_CHECK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->max_smem_optin));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(2 * h->num_sms));
  cfg.blockDim = dim3(kConvThreads);
  cfg.dynamicSmemBytes = 200 * 1024;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kConvKernels[0][1][3][0], &cfg) != cudaSuccess) {
    (void)cudaGetLastError();
    n = 0;                                   // pairs unavailable: the single-CTA variants are used
  }
  h->max_clusters = std::min(n, h->num_sms / 2);
  h->configured |= YV6_CFG_CONV;
  return YV6_OK;
}

extern "C" int yv6_conv_plan(yv6_handle* h, const yv6_conv_desc* d, int32_t* out8) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h != nullptr && out8 != nullptr, "conv_plan: null argument");
  { const int rc0 = conv_configure(h); if (rc0 != YV6_OK) return rc0; }
  ConvPlan plan;
  int rc = plan_conv(h, d, &plan);
  if (rc != YV6_OK) return rc;
  out8[0] = plan.k.BW;
  out8[1] = plan.k.BH;
  out8[2] = plan.k.BI;
  out8[3] = plan.k.BN;
  out8[4] = plan.k.kb_elems;
  out8[5] = plan.k.stages;
  out8[6] = plan.grid;
  out8[7] = plan.k.num_tiles;
  out8[8] = plan.k.halo;
  out8[9] = (plan.k.halo ? plan.k.a_stages * 100 + plan.k.b_resident : 0) + 10 * plan.k.cpair;
  return YV6_OK;
}

// Host-only twin of yv6_conv_plan: plans against stated device properties instead of a handle, makes no CUDA call.
extern "C" int yv6_conv_plan_host(int num_sms, int max_smem_optin, int max_clusters, const yv6_conv_desc* d, int32_t* out12) {
  YV6_REQUIRE(out12 != nullptr, "conv_plan_host: null argument");
  YV6_REQUIRE(num_sms > 0 && max_smem_optin > 0 && max_clusters >= 0, "conv_plan_host: bad device properties");
  yv6_handle fake;
  memset(&fake, 0, sizeof(fake));
  fake.device = -1;
  fake.num_sms = num_sms;
  fake.max_smem_optin = max_smem_optin;
  fake.max_clusters = max_clusters;
  ConvPlan plan;
  int rc = plan_conv(&fake, d, &plan);
  if (rc != YV6_OK) return rc;
  YV6_REQUIRE(plan.smem_bytes <= (size_t)max_smem_optin, "conv_plan_host: plan needs %zu bytes of shared memory, device offers %d",
              plan.smem_bytes, max_smem_optin);
  out12[0] = plan.k.BW;
  out12[1] = plan.k.BH;
  out12[2] = plan.k.BI;
  out12[3] = plan.k.BN;
  out12[4] = plan.k.kb_elems;
  out12[5] = plan.k.stages;
  out12[6] = plan.grid;
  out12[7] = plan.k.num_tiles;
  out12[8] = plan.k.halo;
  out12[9] = (plan.k.halo ? plan.k.a_stages * 100 + plan.k.b_resident : 0) + 10 * plan.k.cpair;
  out12[10] = (int32_t)plan.smem_bytes;
  out12[11] = kConvThreads;
  return YV6_OK;
}

extern "C" int yv6_conv_fwd(yv6_handle* h, const yv6_conv_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h != nullptr, "conv_fwd: null handle");
  { const int rc0 = conv_configure(h); if (rc0 != YV6_OK) return rc0; }
  ConvPlan plan;
  int rc = plan_conv(h, d, &plan);
  if (rc != YV6_OK) return rc;
  const ConvKParams& k = plan.k;
  YV6_REQUIRE(h->encode_tiled != nullptr, "conv_fwd: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");

  // A: (C, W, H, N, plane) over the input (channel slice of a wider NHWC buffer allowed)
  CUtensorMap tmA, tmB;
  const CUtensorMapDataType operand_type = plan.f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  {
    const uint64_t planes = (d->nsplit == 3) ? 3 : 1;
    cuuint64_t dims[5] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N, planes};
    const uint64_t pix = (uint64_t)d->x_c_total * 2;
    uint64_t plane_stride = (d->nsplit == 3) ? (uint64_t)d->x_plane_stride * 2
                                             : (uint64_t)d->N * d->H * d->W * pix;
    YV6_REQUIRE(plane_stride % 16 == 0, "conv: x_plane_stride must be a multiple of 8 elements");
    cuuint64_t strides[4] = {pix, pix * d->W, pix * d->W * d->H, plane_stride};
    cuuint32_t box[5] = {(cuuint32_t)k.kb_elems, (cuuint32_t)(k.BW * k.stride_w), (cuuint32_t)(k.BH * d->stride),
                         (cuuint32_t)k.BI, 1};
    cuuint32_t estr[5] = {1, (cuuint32_t)k.stride_w, (cuuint32_t)d->stride, 1, 1};
    if (k.halo) {       // one dense box per channel block
      box[1] = (k.halo == 2) ? HaloGeom<true>::W : HaloGeom<false>::W;
      box[2] = (k.halo == 2) ? HaloGeom<true>::H : HaloGeom<false>::H;
      estr[1] = estr[2] = 1;
    }
    CUresult cr = h->encode_tiled(&tmA, operand_type, 5, const_cast<void*>(d->x), dims,
                                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, plan.swz,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      yv6_set_error("conv: cuTensorMapEncodeTiled(A) failed with %d (C=%d W=%d H=%d N=%d box=%u,%u,%u,%u)", (int)cr,
                    d->Cin, d->W, d->H, d->N, box[0], box[1], box[2], box[3]);
      return YV6_ERR_CUDA;
    }
  }
  {
    const uint64_t planes = (d->nsplit == 3) ? 3 : 1;
    const uint64_t ktot = (uint64_t)k.taps * d->Cin;
    cuuint64_t dims[3] = {ktot, (cuuint64_t)d->Cout, planes};
    uint64_t plane_stride = (d->nsplit == 3) ? (uint64_t)d->w_plane_stride * 2 : ktot * 2 * d->Cout;
    YV6_REQUIRE(plane_stride % 16 == 0, "conv: w_plane_stride must be a multiple of 8 elements");
    cuuint64_t strides[2] = {ktot * 2, plane_stride};
    cuuint32_t box[3] = {(cuuint32_t)k.kb_elems, (cuuint32_t)k.b_rows, 1};   // pair mode: each CTA loads half of the N tile
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult cr = h->encode_tiled(&tmB, operand_type, 3, const_cast<void*>(d->w), dims,
                                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, plan.swz,
                                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      yv6_set_error("conv: cuTensorMapEncodeTiled(B) failed with %d", (int)cr);
      return YV6_ERR_CUDA;
    }
  }
  // Y: (C, W, H, N) over the destination view, for the TMA-store epilogue (unused, left zero, otherwise)
  CUtensorMap tmY;
  memset(&tmY, 0, sizeof(tmY));
  if (k.tma_store) {
    const bool f32 = d->y_dtype == YV6_DT_F32;
    const uint64_t esz = f32 ? 4 : 2;
    cuuint64_t dims[4] = {(cuuint64_t)d->Cout, (cuuint64_t)k.Wo, (cuuint64_t)k.Ho, (cuuint64_t)d->N};
    cuuint64_t strides[3] = {(cuuint64_t)d->y_w_stride * esz, (cuuint64_t)d->y_h_stride * esz, (cuuint64_t)d->y_img_stride * esz};
    const int box_bytes = y_box_bytes(k.BN, (int)esz);
    cuuint32_t box[4] = {(cuuint32_t)(box_bytes / esz), (cuuint32_t)k.BW, (cuuint32_t)(f32 ? k.BH / 2 : k.BH), (cuuint32_t)k.BI};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult cr = h->encode_tiled(&tmY, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : operand_type, 4, d->y, dims,
                                  strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                  box_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      yv6_set_error("conv: cuTensorMapEncodeTiled(Y) failed with %d (C=%d W=%d H=%d N=%d strides=%lld,%lld,%lld)", (int)cr, d->Cout,
                    k.Wo, k.Ho, d->N, (long long)d->y_w_stride, (long long)d->y_h_stride, (long long)d->y_img_stride);
      return YV6_ERR_CUDA;
    }
  }

  const int mode = k.halo ? (k.halo == 2 ? 3 : 1) + (k.b_resident ? 1 : 0) : 0;
  const int bn_idx = k.BN == 32 ? 0 : k.BN == 64 ? 1 : k.BN == 96 ? 2 : 3;
  ConvKernelFn fn = kConvKernels[plan.f16][k.cpair][bn_idx][mode];
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)plan.grid);
  cfg.blockDim = dim3((unsigned)kConvThreads);
  cfg.dynamicSmemBytes = plan.smem_bytes;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  if (k.cpair) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  YV6_CHECK_CUDA(cudaLaunchKernelEx(&cfg, fn, tmA, tmB, tmY, k));
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
