// yv6_augment.cu -- the pixels of TrainValDataset.__getitem__ (yolov6/data/datasets.py:166-255) with augment=True, for a
// whole batch in two launches:
//   yv6_aug_resize: load_image's cv2.resize INTER_LINEAR (datasets.py:287-295) of every source, and (second launch) the
//                   letterbox branch's resize of those results (data_augment.py:52-53);
//   yv6_aug_resize_frames: the same resize from frames anywhere in device memory (yv6_lb_src records: a decoder's
//                   output, a crop view, the device frame cache), into packed BGR HWC in the arena;
//   yv6_augment:    mosaic / letterbox canvas + random_affine's cv2.warpAffine, mixup, augment_hsv, flips, HWC BGR ->
//                   CHW RGB, written straight into the training input.
//
// warpAffine is OpenCV's uint8 INTER_LINEAR / BORDER_CONSTANT path: with the inverted matrix m (host, double),
//   X = (rint((m1 * y + m2) * 1024) + 16 + rint(m0 * x * 1024)) >> 5   (and Y with m4, m5, m3),
// integer tap X >> 5, 5-bit fraction X & 31, the 32 x 32 bilinear table (entries (32 - f) * (32 - g) * 32 etc., exact
// integers), (sum + 2^14) >> 15, and a tap outside the canvas reads 114.  The canvas is never materialised: its pixels
// are copies of the resized sources, so sampling the placed rectangles gives the same bytes as the reference's img4.
//
// HSV: BGR -> HSV is OpenCV's 12-bit fixed point (sdiv = rint((255 << 12) / i), hdiv = rint((180 << 12) / (6 i)));
// HSV -> BGR is its AVX2 float path: s, v scaled by 1/255, h by 6/180, tab2 = v * fma(-s, f, 1), tab3 = v * fma(-s, 1 - f,
// 1), times 255, truncated.  Every float / double operation is an explicit intrinsic, so ptxas cannot contract it
// (the two fmas are OpenCV's own).
#include "yv6_common.cuh"
#include "yv6_frame_src.cuh"
#include "yv6_handle.h"
#include "yv6_resize.cuh"

namespace yv6 {

constexpr int kAugPix = 16;     // output pixels per thread: one 16-byte store into each channel plane

// Job j resizes its source to nh x nw packed BGR HWC at base + dst_off.  The source is read through srcs[j]
// (yv6_aug_resize_frames: any frame in device memory, either layout) or, when srcs is null, as packed BGR HWC at
// base + src_off (yv6_aug_resize): only the address of a tap depends on the record.
__global__ void __launch_bounds__(256) aug_resize_kernel(const yv6_lb_src* __restrict__ srcs, uint8_t* __restrict__ base,
                                                         const int64_t* __restrict__ jobs) {
  const int64_t* j = jobs + (int64_t)blockIdx.y * YV6_AUG_JOB;
  const int64_t src_off = j[0], dst_off = j[3];
  const int h0 = (int)j[1], w0 = (int)j[2], nh = (int)j[4], nw = (int)j[5];
  int64_t row_pitch, ch[3];
  int px;
  const uint8_t* im = frame_source(srcs, blockIdx.y, srcs ? nullptr : base + src_off, w0, row_pitch, px, ch);
  uint8_t* out = base + dst_off;
  const double sy = lin_scale(nh, h0), sx = lin_scale(nw, w0);
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < (int64_t)nh * nw; p += (int64_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / nw), x = (int)(p - (int64_t)y * nw);
    uint8_t* o = out + p * 3;
    if (nh == h0 && nw == w0) {                // cv2.resize to the same size copies (and here converts the layout)
      const uint8_t* s = im + (int64_t)y * row_pitch + (int64_t)x * px;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = __ldg(s + ch[2 - c]);     // output channel c (B, G, R) is canvas channel 2 - c
      continue;
    }
    const LinTap v = lin_tap(y, sy, h0, false);
    const LinTap hz = lin_tap(x, sx, w0, true);
    const uint8_t* r0 = im + (int64_t)v.s0 * row_pitch;
    const uint8_t* r1 = im + (int64_t)v.s1 * row_pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = lin_pixel(r0 + ch[2 - c], r1 + ch[2 - c], v, hz, 0, px);
  }
}

// Canvas pixel (y, x) of canvas k, BGR into px.
__device__ __forceinline__ void canvas_px(const uint8_t* __restrict__ base, const yv6_aug_sample& s, int k, int y, int x, int px[3]) {
  px[0] = px[1] = px[2] = 114;
  if (y < 0 || x < 0 || y >= s.ch[k] || x >= s.cw[k]) return;
  for (int t = s.ntile[k] - 1; t >= 0; --t) {
    const yv6_aug_tile& tl = s.tile[k][t];
    if (y >= tl.y0 && y < tl.y1 && x >= tl.x0 && x < tl.x1) {
      const uint8_t* p = base + tl.org + ((int64_t)y * tl.pitch + x) * 3;
      px[0] = __ldg(p), px[1] = __ldg(p + 1), px[2] = __ldg(p + 2);
      return;
    }
  }
}

// cv2.warpAffine's INTER_LINEAR sample of canvas k at output pixel (y, x).
__device__ __forceinline__ void warp_px(const uint8_t* __restrict__ base, const yv6_aug_sample& s, int k, int y, int x, int out[3]) {
  const double* m = s.minv[k];
  const int X = (__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), 1024.0)) + 16 +
                 __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)x), 1024.0))) >> 5;
  const int Y = (__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), 1024.0)) + 16 +
                 __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)x), 1024.0))) >> 5;
  const int sx = X >> 5, fx = X & 31, sy = Y >> 5, fy = Y & 31;
  const int w00 = (32 - fx) * (32 - fy) * 32, w01 = fx * (32 - fy) * 32, w10 = (32 - fx) * fy * 32, w11 = fx * fy * 32;
  int a[3], b[3], c[3], d[3];
  canvas_px(base, s, k, sy, sx, a);
  canvas_px(base, s, k, sy, sx + 1, b);
  canvas_px(base, s, k, sy + 1, sx, c);
  canvas_px(base, s, k, sy + 1, sx + 1, d);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) out[ch] = min(max((a[ch] * w00 + b[ch] * w01 + c[ch] * w10 + d[ch] * w11 + (1 << 14)) >> 15, 0), 255);
}

// augment_hsv's cvtColor(BGR2HSV) -> LUT -> cvtColor(HSV2BGR) of one BGR pixel, in place.
__device__ __forceinline__ void hsv_px(int p[3], const uint8_t* lut, const int* sdiv, const int* hdiv) {
  const int b = p[0], g = p[1], r = p[2];
  const int v = max(max(b, g), r);
  const int diff = v - min(min(b, g), r);
  const int s = (diff * sdiv[v] + (1 << 11)) >> 12;
  int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv[diff] + (1 << 11)) >> 12;
  if (h < 0) h += 180;
  const float hf = __fmul_rn((float)lut[h], 6.0f / 180.0f);
  const float sf = __fmul_rn((float)lut[256 + s], 1.0f / 255.0f);
  const float vf = __fmul_rn((float)lut[512 + v], 1.0f / 255.0f);
  const float pre = truncf(hf);
  const float f = __fsub_rn(hf, pre);
  const int sector = (int)pre % 6;
  float tab[4];
  tab[0] = vf;
  tab[1] = __fmul_rn(vf, __fsub_rn(1.f, sf));
  tab[2] = __fmul_rn(vf, __fmaf_rn(-sf, f, 1.f));
  tab[3] = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.f, f), 1.f));
  const int i0[6] = {1, 1, 3, 0, 0, 2}, i1[6] = {3, 0, 0, 2, 1, 1}, i2[6] = {0, 2, 1, 1, 3, 0};
  p[0] = __float2int_rz(__fmul_rn(tab[i0[sector]], 255.f));
  p[1] = __float2int_rz(__fmul_rn(tab[i1[sector]], 255.f));
  p[2] = __float2int_rz(__fmul_rn(tab[i2[sector]], 255.f));
}

// thread = 16 consecutive output pixels of one row of one image.
__global__ void __launch_bounds__(128) augment_kernel(const uint8_t* __restrict__ base, const yv6_aug_sample* __restrict__ samples,
                                                      int H, int W, uint8_t* __restrict__ dst) {
  __shared__ int sdiv[256], hdiv[256];
  __shared__ uint8_t lut[3 * 256];
  const int b = blockIdx.y;
  const yv6_aug_sample& s = samples[b];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    sdiv[i] = i ? __double2int_rn(__ddiv_rn((double)(255 << 12), (double)i)) : 0;
    hdiv[i] = i ? __double2int_rn(__ddiv_rn((double)(180 << 12), __dmul_rn(6.0, (double)i))) : 0;
  }
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i] = s.lut[i / 256][i % 256];
  __syncthreads();
  const int per_row = W / kAugPix;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * per_row) return;
  const int y = q / per_row, x0 = (q - y * per_row) * kAugPix;
  const int py = s.flipud ? H - 1 - y : y;
  alignas(16) uint8_t o[3][kAugPix];
#pragma unroll 1
  for (int i = 0; i < kAugPix; ++i) {
    const int px = s.fliplr ? W - 1 - (x0 + i) : x0 + i;
    int p[3];
    warp_px(base, s, 0, py, px, p);
    if (s.mixup) {
      int p2[3];
      warp_px(base, s, 1, py, px, p2);
      const double r = s.mix_r, r1 = __dsub_rn(1.0, r);
#pragma unroll
      for (int c = 0; c < 3; ++c) p[c] = __double2int_rz(__dadd_rn(__dmul_rn((double)p[c], r), __dmul_rn((double)p2[c], r1)));
    }
    if (s.hsv) hsv_px(p, lut, sdiv, hdiv);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c][i] = (uint8_t)p[2 - c];          // BGR -> RGB
  }
  const int64_t plane = (int64_t)H * W;
  uint8_t* d = dst + (int64_t)b * 3 * plane + (int64_t)y * W + x0;
#pragma unroll
  for (int c = 0; c < 3; ++c) *reinterpret_cast<uint4*>(d + c * plane) = *reinterpret_cast<const uint4*>(o[c]);
}

}  // namespace yv6

using namespace yv6;

static int launch_aug_resize(const yv6_lb_src* srcs, uint8_t* base, const int64_t* jobs, int32_t J, int64_t max_pix, void* stream) {
  YV6_REQUIRE(J <= 65535, "aug_resize: %d jobs exceed one launch", J);
  if (J == 0 || max_pix == 0) return YV6_OK;
  const int64_t blocks = (max_pix + 255) / 256;
  aug_resize_kernel<<<dim3((unsigned)(blocks < 1024 ? blocks : 1024), J), 256, 0, (cudaStream_t)stream>>>(srcs, base, jobs);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_aug_resize(yv6_handle* h, uint8_t* base, const int64_t* jobs, int32_t J, int64_t max_pix, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && base && jobs && J >= 0 && max_pix >= 0, "aug_resize: bad argument");
  return launch_aug_resize(nullptr, base, jobs, J, max_pix, stream);
}

extern "C" int yv6_aug_resize_frames(yv6_handle* h, const yv6_lb_src* srcs, const int64_t* jobs, int32_t J, int64_t max_pix,
                                     uint8_t* base, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && srcs && base && jobs && J >= 0 && max_pix >= 0, "aug_resize_frames: bad argument");
  return launch_aug_resize(srcs, base, jobs, J, max_pix, stream);
}

extern "C" int yv6_augment(yv6_handle* h, const uint8_t* base, const yv6_aug_sample* samples, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                           void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && base && samples && dst && B > 0 && H > 0 && W > 0, "augment: bad argument");
  YV6_REQUIRE(W % 32 == 0 && ((uintptr_t)dst & 15) == 0, "augment: W (%d) must be a multiple of 32 and dst 16-byte aligned", W);
  YV6_REQUIRE(B <= 65535, "augment: batch %d too large", B);
  const int chunks = H * (W / kAugPix);
  augment_kernel<<<dim3((chunks + 127) / 128, B), 128, 0, (cudaStream_t)stream>>>(base, samples, H, W, dst);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
