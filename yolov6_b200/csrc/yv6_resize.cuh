// yv6_resize.cuh -- one axis of OpenCV's uint8 INTER_LINEAR cv2.resize, shared by yv6_letterbox.cu and yv6_augment.cu.
// The rule (see yv6_letterbox.cu for why each part matters): source coordinate in double from the inverted inverse scale,
// 11-bit coefficients, horizontal border taps clamped with a zero fraction, vertical rows clamped with the unreset fraction,
// and the truncating vertical pass of OpenCV's SIMD kernel.  Every channel is resized on its own, so the layout of the
// channels changes only the address of a tap.
#pragma once
#include <cstdint>

namespace yv6 {

struct LinTap {
  int s0, s1, c0, c1;
};

// One axis of cv::resize's INTER_LINEAR coefficient table for destination index d.
__device__ __forceinline__ LinTap lin_tap(int d, double scale, int src, bool reset_border) {
  const float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int s = (int)floorf(f);
  float fr = __fsub_rn(f, (float)s);
  if (reset_border) {
    if (s < 0) fr = 0.f, s = 0;
    if (s >= src - 1) fr = 0.f, s = src - 1;
  }
  LinTap t;
  t.c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fr), 2048.f));
  t.c1 = __float2int_rn(__fmul_rn(fr, 2048.f));
  t.s0 = min(max(s, 0), src - 1);
  t.s1 = min(max(s + 1, 0), src - 1);
  return t;
}

// cv::resize keeps the inverse scale and inverts it: the per-axis scale of an n0 -> n resize.
__device__ __forceinline__ double lin_scale(int n, int n0) { return __ddiv_rn(1.0, __ddiv_rn((double)n, (double)n0)); }

// One channel of the resized pixel from the two vertical taps' rows r0, r1 and horizontal tap hz: the channel's byte of
// pixel x lies at r + x * px + ch (px = 3 for uint8 HWC with 3 channels, px = 1 for one plane of CHW).
__device__ __forceinline__ uint8_t lin_pixel(const uint8_t* r0, const uint8_t* r1, const LinTap& v, const LinTap& hz, int ch,
                                             int px = 3) {
  const int S0 = __ldg(r0 + hz.s0 * px + ch) * hz.c0 + __ldg(r0 + hz.s1 * px + ch) * hz.c1;
  const int S1 = __ldg(r1 + hz.s0 * px + ch) * hz.c0 + __ldg(r1 + hz.s1 * px + ch) * hz.c1;
  const int t = (((v.c0 * (S0 >> 4)) >> 16) + ((v.c1 * (S1 >> 4)) >> 16) + 2) >> 2;
  return (uint8_t)min(max(t, 0), 255);
}

}  // namespace yv6
