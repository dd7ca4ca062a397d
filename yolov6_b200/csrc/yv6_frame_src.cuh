// yv6_frame_src.cuh -- where the pixels of a decoded frame lie, shared by every kernel that reads frames through a
// yv6_lb_src record (yv6_letterbox.cu, yv6_augment.cu).
#pragma once
#include <cstdint>

#include "../../include/yv6.h"

namespace yv6 {

// Image b lies at srcs[b] or, when srcs is null, at `packed` as BGR HWC with rows of w0 * 3 bytes.  Canvas channel c
// (R, G, B) of pixel x of a row lies at row + x * px + ch[c]: BGR HWC reads channel 2 - c, RGB CHW plane c.
__device__ __forceinline__ const uint8_t* frame_source(const yv6_lb_src* srcs, int b, const uint8_t* packed, int w0,
                                                       int64_t& row_pitch, int& px, int64_t (&ch)[3]) {
  const uint8_t* im;
  int64_t plane_pitch;
  int layout;
  if (srcs) {
    const yv6_lb_src s = srcs[b];
    im = s.base, row_pitch = s.row_pitch, plane_pitch = s.plane_pitch, layout = s.layout;
  } else {
    im = packed, row_pitch = (int64_t)w0 * 3, plane_pitch = 0, layout = YV6_LB_BGR_HWC;
  }
  const bool chw = layout == YV6_LB_RGB_CHW;
  px = chw ? 1 : 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) ch[c] = chw ? c * plane_pitch : 2 - c;
  return im;
}

}  // namespace yv6
