// yv6_letterbox.cu -- the image side of the reference's Inferer around the model, for a whole batch per launch:
//   yv6_letterbox:      letterbox (yolov6/data/data_augment.py:29-58, auto=False) + HWC->CHW + BGR->RGB of
//                       Inferer.process_image (core/inferer.py:161-171); the 1/255 stays in the stem kernel.
//   yv6_letterbox_frames: the same canvases from images anywhere in device memory, each addressed by a yv6_lb_src record
//                       (BGR HWC with padded rows, or RGB CHW as torchvision's decoders return it).
//   yv6_letterbox_val:  the Evaler's validation images (TrainValDataset with augment=False): load_image's resize --
//                       cv2.INTER_AREA when it shrinks, INTER_LINEAR when it enlarges -- then letterbox(auto=False,
//                       scaleup=False) onto the batch canvas, which never resizes again, + HWC->CHW + BGR->RGB.
//   yv6_rescale_boxes:  Inferer.rescale (core/inferer.py:173-188) followed by the `.round()` of inferer.py:103.
//
// Resampling is OpenCV's uint8 INTER_LINEAR path of cv2.resize, reproduced bit for bit:
//   - source coordinate fx = (float)((dx + 0.5) * scale - 0.5) in DOUBLE, scale = 1 / (dst / src) (cv::resize keeps the
//     inverse scale and inverts it), sx = floor(fx), fx -= sx in float;
//   - horizontal: a border tap (sx < 0 or sx >= w0 - 1) is clamped AND gets fx = 0; coefficients
//     saturate_cast<short>((1 - fx) * 2048), saturate_cast<short>(fx * 2048) (round half to even); S = s0*a0 + s1*a1;
//   - vertical: the row indices sy, sy + 1 are clamped to [0, h0) but fy is NOT reset at the borders, so an upscaled
//     image's first / last rows blend one row with itself at uneven weights -- which the truncating vertical pass below
//     does not always map back to that row's value;
//   - vertical pass of the SIMD kernel (VResizeLinearVec_32s8u): ((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2.
// The double-precision coordinate and the unreset vertical fraction are what a float32 restatement with clamped fy gets
// wrong on upscaling shapes.  Every float / double operation is an explicit round-to-nearest intrinsic, so ptxas cannot
// contract it into an FMA.
#include "yv6_common.cuh"
#include "yv6_frame_src.cuh"
#include "yv6_handle.h"
#include "yv6_resize.cuh"

namespace yv6 {

constexpr int kLbPix = 16;     // output pixels per thread: one 16-byte store into each channel plane

// geo [B][YV6_LB_GEO] = (src_off, h0, w0, nh, nw, top, left, 0); thread = 16 consecutive pixels of one canvas row.
// Image b is read through srcs[b] (yv6_letterbox_frames) or, when srcs is null, as packed BGR HWC at packed + src_off
// (yv6_letterbox): one sampling routine for both entry points, only the address of a tap depends on the record.
__global__ void __launch_bounds__(256) letterbox_kernel(const yv6_lb_src* __restrict__ srcs, const uint8_t* __restrict__ packed,
                                                        const int32_t* __restrict__ geo, int H, int W, uint8_t* __restrict__ dst) {
  const int b = blockIdx.y;
  const int per_row = W / kLbPix;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * per_row) return;
  const int y = q / per_row, x0 = (q - y * per_row) * kLbPix;
  const int32_t* g = geo + b * YV6_LB_GEO;
  const int h0 = __ldg(g + 1), w0 = __ldg(g + 2), nh = __ldg(g + 3), nw = __ldg(g + 4), top = __ldg(g + 5), left = __ldg(g + 6);
  int64_t row_pitch, ch[3];
  int px;
  const uint8_t* im = frame_source(srcs, b, srcs ? nullptr : packed + __ldg(g + 0), w0, row_pitch, px, ch);
  alignas(16) uint8_t o[3][kLbPix];
  const int ys = y - top;
  if (ys < 0 || ys >= nh) {
#pragma unroll
    for (int i = 0; i < kLbPix; ++i) o[0][i] = o[1][i] = o[2][i] = 114;
  } else if (nh == h0 && nw == w0) {           // data_augment.py:52: no resize, a plain copy
    const uint8_t* row = im + (int64_t)ys * row_pitch;
#pragma unroll
    for (int i = 0; i < kLbPix; ++i) {
      const int xs = x0 + i - left;
      const bool in = xs >= 0 && xs < nw;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c][i] = in ? __ldg(row + ch[c] + xs * px) : (uint8_t)114;
    }
  } else {
    const double sy_scale = lin_scale(nh, h0);
    const double sx_scale = lin_scale(nw, w0);
    const LinTap v = lin_tap(ys, sy_scale, h0, false);
    const uint8_t* r0 = im + (int64_t)v.s0 * row_pitch;
    const uint8_t* r1 = im + (int64_t)v.s1 * row_pitch;
#pragma unroll
    for (int i = 0; i < kLbPix; ++i) {
      const int xs = x0 + i - left;
      if (xs < 0 || xs >= nw) {
        o[0][i] = o[1][i] = o[2][i] = 114;
        continue;
      }
      const LinTap hz = lin_tap(xs, sx_scale, w0, true);
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c][i] = lin_pixel(r0 + ch[c], r1 + ch[c], v, hz, 0, px);
    }
  }
  const int64_t plane = (int64_t)H * W;
  uint8_t* d = dst + (int64_t)b * 3 * plane + (int64_t)y * W + x0;
#pragma unroll
  for (int c = 0; c < 3; ++c) *reinterpret_cast<uint4*>(d + c * plane) = *reinterpret_cast<const uint4*>(o[c]);
}

constexpr int kValPix = 4;     // yv6_letterbox_val: output pixels per thread, one 4-byte store into each channel plane

// One axis of OpenCV's computeResizeAreaTab (resize.cpp) for destination index d of an n0 -> n shrink, scale = n0 / n as
// cv::resize forms it: the taps are [sx1 - 1 when left] sx1 .. sx2 - 1 [sx2 when right], in that (source) order, with
// weights a_left, a_mid each, a_right.  Double arithmetic as OpenCV's, each weight rounded to float once.
struct AreaAxis {
  int sx1, sx2;
  bool left, right;
  float a_left, a_mid, a_right;
};

__device__ __forceinline__ AreaAxis area_axis(int d, double scale, int n0) {
  const double f1 = __dmul_rn((double)d, scale), f2 = __dadd_rn(f1, scale);
  const double cell = fmin(scale, __dsub_rn((double)n0, f1));
  AreaAxis a;
  a.sx2 = min((int)floor(f2), n0 - 1);
  a.sx1 = min((int)ceil(f1), a.sx2);
  const double l = __dsub_rn((double)a.sx1, f1), r = __dsub_rn(f2, (double)a.sx2);
  a.left = l > 1e-3;
  a.right = r > 1e-3;
  a.a_left = __double2float_rn(__ddiv_rn(l, cell));
  a.a_mid = __double2float_rn(__ddiv_rn(1.0, cell));
  a.a_right = __double2float_rn(__ddiv_rn(fmin(fmin(r, 1.0), cell), cell));
  return a;
}

// Source tap t (0-based) of an axis and its weight.
__device__ __forceinline__ int area_tap(const AreaAxis& a, int t, float& w) {
  if (a.left) {
    if (t == 0) return w = a.a_left, a.sx1 - 1;
    --t;
  }
  const int s = a.sx1 + t;
  w = s < a.sx2 ? a.a_mid : a.a_right;
  return s;
}

__device__ __forceinline__ int area_taps(const AreaAxis& a) { return (a.sx2 - a.sx1) + a.left + a.right; }

// geo [B][YV6_LB_GEO] = (src_off, h0, w0, nh, nw, top, left, mode), mode YV6_VAL_*: the image of load_image (copy,
// INTER_LINEAR upscale, INTER_AREA shrink) placed at (top, left) of the batch canvas; thread = 16 pixels of one canvas row.
//   AREA (resizeArea_): per destination row, for each source row sy of its vertical taps (weight beta), the float sum over
//     the horizontal taps of S * alpha, then sum = beta * buf for the first row and sum += beta * buf after; the result is
//     saturate_cast<uchar> (round half to even).  Each product and sum is one float operation in OpenCV's order.
//   AREA_FAST (resizeAreaFast_, both scales integers): the int sum of the sx x sy box, (sum + 2) >> 2 for 2 x 2
//     (ResizeAreaFastVec), otherwise saturate_cast<uchar>(sum * (1.f / area)).
__global__ void __launch_bounds__(256) letterbox_val_kernel(const yv6_lb_src* __restrict__ srcs, const int32_t* __restrict__ geo,
                                                            int H, int W, uint8_t* __restrict__ dst) {
  const int b = blockIdx.y;
  const int per_row = W / kValPix;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * per_row) return;
  const int y = q / per_row, x0 = (q - y * per_row) * kValPix;
  const int32_t* g = geo + b * YV6_LB_GEO;
  const int h0 = __ldg(g + 1), w0 = __ldg(g + 2), nh = __ldg(g + 3), nw = __ldg(g + 4), top = __ldg(g + 5), left = __ldg(g + 6);
  const int mode = __ldg(g + 7);
  alignas(4) uint8_t o[3][kValPix];
#pragma unroll
  for (int i = 0; i < kValPix; ++i) o[0][i] = o[1][i] = o[2][i] = 114;
  const int ys = y - top;
  if (ys >= 0 && ys < nh) {
    int64_t row_pitch, ch[3];
    int px;
    const uint8_t* im = frame_source(srcs, b, nullptr, w0, row_pitch, px, ch);
    const int xa = left - x0, xb = left + nw - x0;      // canvas pixels x0 + [xa, xb) hold the image
    if (mode == YV6_VAL_COPY) {
      const uint8_t* row = im + (int64_t)ys * row_pitch;
      #pragma unroll
      for (int i = 0; i < kValPix; ++i) {
        if (i < xa || i >= xb) continue;
        const int xs = x0 + i - left;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c][i] = __ldg(row + ch[c] + xs * px);
      }
    } else if (mode == YV6_VAL_LINEAR) {
      const LinTap v = lin_tap(ys, lin_scale(nh, h0), h0, false);
      const double sx_scale = lin_scale(nw, w0);
      const uint8_t* r0 = im + (int64_t)v.s0 * row_pitch;
      const uint8_t* r1 = im + (int64_t)v.s1 * row_pitch;
      #pragma unroll
      for (int i = 0; i < kValPix; ++i) {
        if (i < xa || i >= xb) continue;
        const LinTap hz = lin_tap(x0 + i - left, sx_scale, w0, true);
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c][i] = lin_pixel(r0 + ch[c], r1 + ch[c], v, hz, 0, px);
      }
    } else if (mode == YV6_VAL_AREA_FAST) {
      const int kx = w0 / nw, ky = h0 / nh;
      const float inv = __fdiv_rn(1.f, (float)(kx * ky));
      const uint8_t* r0 = im + (int64_t)(ys * ky) * row_pitch;
      #pragma unroll
      for (int i = 0; i < kValPix; ++i) {
        if (i < xa || i >= xb) continue;
        const int sx0 = (x0 + i - left) * kx;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          int sum = 0;
          for (int dy = 0; dy < ky; ++dy) {
            const uint8_t* r = r0 + dy * row_pitch + ch[c];
            for (int dx = 0; dx < kx; ++dx) sum += __ldg(r + (int64_t)(sx0 + dx) * px);
          }
          o[c][i] = (uint8_t)(kx == 2 && ky == 2 ? (sum + 2) >> 2 : min(__float2int_rn(__fmul_rn((float)sum, inv)), 255));
        }
      }
    } else {
      const AreaAxis va = area_axis(ys, lin_scale(nh, h0), h0);
      const double sx_scale = lin_scale(nw, w0);
      const int nv = area_taps(va);
      #pragma unroll
      for (int i = 0; i < kValPix; ++i) {
        if (i < xa || i >= xb) continue;
        const AreaAxis ha = area_axis(x0 + i - left, sx_scale, w0);
        const int nhz = area_taps(ha);
        float acc[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < nv; ++j) {
          float beta;
          const uint8_t* r = im + (int64_t)area_tap(va, j, beta) * row_pitch;
          float buf[3] = {0.f, 0.f, 0.f};
          for (int k = 0; k < nhz; ++k) {
            float alpha;
            const int64_t sx = (int64_t)area_tap(ha, k, alpha) * px;
#pragma unroll
            for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)__ldg(r + ch[c] + sx), alpha));
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[c] = j == 0 ? __fmul_rn(beta, buf[c]) : __fadd_rn(acc[c], __fmul_rn(beta, buf[c]));
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c][i] = (uint8_t)min(max(__float2int_rn(acc[c]), 0), 255);
      }
    }
  }
  const int64_t plane = (int64_t)H * W;
  uint8_t* d = dst + (int64_t)b * 3 * plane + (int64_t)y * W + x0;
#pragma unroll
  for (int c = 0; c < 3; ++c) *reinterpret_cast<uint32_t*>(d + c * plane) = *reinterpret_cast<const uint32_t*>(o[c]);
}

// Inferer.rescale(img.shape[2:], det[:, :4], img_src.shape).round(): ratio and padding are the reference's Python doubles,
// the box arithmetic is torch's fp32 (x - (float)pad) / (float)ratio, clamp to the source image, round half to even.
// Rows beyond count[b] are zeroed.
__global__ void rescale_boxes_kernel(const float* __restrict__ det, const int32_t* __restrict__ count, const int32_t* __restrict__ geo,
                                     int B, int max_det, int H, int W, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * max_det) return;
  const int b = i / max_det, j = i - b * max_det;
  float* o = out + (int64_t)i * 6;
  if (j >= count[b]) {
    o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0.f;
    return;
  }
  const double h0 = geo[b * YV6_LB_GEO + 1], w0 = geo[b * YV6_LB_GEO + 2];
  const double ratio = fmin(__ddiv_rn((double)H, h0), __ddiv_rn((double)W, w0));                 // inferer.py:176
  const float pad_x = __double2float_rn(__ddiv_rn(__dsub_rn((double)W, __dmul_rn(w0, ratio)), 2.0));   // :177
  const float pad_y = __double2float_rn(__ddiv_rn(__dsub_rn((double)H, __dmul_rn(h0, ratio)), 2.0));
  const float rf = __double2float_rn(ratio), wf = (float)w0, hf = (float)h0;
  const float* r = det + (int64_t)i * 6;
  o[0] = rintf(fminf(fmaxf(__fdiv_rn(__fsub_rn(r[0], pad_x), rf), 0.f), wf));
  o[1] = rintf(fminf(fmaxf(__fdiv_rn(__fsub_rn(r[1], pad_y), rf), 0.f), hf));
  o[2] = rintf(fminf(fmaxf(__fdiv_rn(__fsub_rn(r[2], pad_x), rf), 0.f), wf));
  o[3] = rintf(fminf(fmaxf(__fdiv_rn(__fsub_rn(r[3], pad_y), rf), 0.f), hf));
  o[4] = r[4];
  o[5] = r[5];
}

}  // namespace yv6

using namespace yv6;

static int launch_letterbox(const yv6_lb_src* srcs, const uint8_t* packed, const int32_t* geo, int32_t B, int32_t H, int32_t W,
                            uint8_t* dst, void* stream) {
  YV6_REQUIRE(W % kLbPix == 0 && ((uintptr_t)dst & 15) == 0, "letterbox: W (%d) must be a multiple of 16 and dst 16-byte aligned", W);
  YV6_REQUIRE(B <= 65535, "letterbox: batch %d too large", B);
  const int chunks = H * (W / kLbPix);
  letterbox_kernel<<<dim3((chunks + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(srcs, packed, geo, H, W, dst);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_letterbox(yv6_handle* h, const uint8_t* src, const int32_t* geo, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                             void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && src && geo && dst && B > 0 && H > 0 && W > 0, "letterbox: bad argument");
  return launch_letterbox(nullptr, src, geo, B, H, W, dst, stream);
}

extern "C" int yv6_letterbox_frames(yv6_handle* h, const yv6_lb_src* srcs, const int32_t* geo, int32_t B, int32_t H, int32_t W,
                                    uint8_t* dst, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && srcs && geo && dst && B > 0 && H > 0 && W > 0, "letterbox_frames: bad argument");
  return launch_letterbox(srcs, nullptr, geo, B, H, W, dst, stream);
}

extern "C" int yv6_letterbox_val(yv6_handle* h, const yv6_lb_src* srcs, const int32_t* geo, int32_t B, int32_t H, int32_t W, uint8_t* dst,
                                 void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && srcs && geo && dst && B > 0 && H > 0 && W > 0, "letterbox_val: bad argument");
  YV6_REQUIRE(W % kLbPix == 0 && ((uintptr_t)dst & 15) == 0, "letterbox_val: W (%d) must be a multiple of 16 and dst 16-byte aligned", W);
  YV6_REQUIRE(B <= 65535, "letterbox_val: batch %d too large", B);
  const int chunks = H * (W / kValPix);
  letterbox_val_kernel<<<dim3((chunks + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(srcs, geo, H, W, dst);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_rescale_boxes(yv6_handle* h, const float* det, const int32_t* count, const int32_t* geo, int32_t B, int32_t max_det,
                                 int32_t H, int32_t W, float* out, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && det && count && geo && out && B > 0 && max_det > 0 && H > 0 && W > 0, "rescale_boxes: bad argument");
  const int total = B * max_det;
  rescale_boxes_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(det, count, geo, B, max_det, H, W, out);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
