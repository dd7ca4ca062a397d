// yv6_scale_coords.cuh -- Evaler.scale_coords (yolov6/core/evaler.py:340-359) on one xyxy box, shared by the evaluation
// post-processing (yv6_nms.cu), the PR-metric matching (yv6_metrics.cu) and the COCO box evaluation (yv6_cocoeval.cu).  fp32 in the reference's operation order with
// explicit round-to-nearest ops, so the boxes are bit-identical to the reference's:
//   x -= pad_x; x /= gain_w; clamp(0, w0)   (same for y with pad_y / gain_h / h0)
// m [6] = (gain_h, gain_w, pad_x, pad_y, h0, w0): one row of evalpost.image_meta.
#pragma once
#include <cuda_runtime.h>

namespace yv6 {

__device__ __forceinline__ float4 scale_coords_rn(float x1, float y1, float x2, float y2, const float* __restrict__ m) {
  const float gh = m[0], gw = m[1], px = m[2], py = m[3], h0 = m[4], w0 = m[5];
  return make_float4(fminf(fmaxf(__fdiv_rn(__fsub_rn(x1, px), gw), 0.f), w0), fminf(fmaxf(__fdiv_rn(__fsub_rn(y1, py), gh), 0.f), h0),
                     fminf(fmaxf(__fdiv_rn(__fsub_rn(x2, px), gw), 0.f), w0), fminf(fmaxf(__fdiv_rn(__fsub_rn(y2, py), gh), 0.f), h0));
}

// the rest of Evaler.convert_to_coco_format (evaler.py:331-338, 369-370) on a scaled box: box_convert to centre form, then the
// shift of the centre to the top-left corner -> (x_tl, y_tl, w, h)
//   xc = (x1 + x2) / 2; w = x2 - x1; x_tl = xc - w / 2
__device__ __forceinline__ float4 coco_xywh_rn(float4 s) {
  const float xc = __fdiv_rn(__fadd_rn(s.x, s.z), 2.f), yc = __fdiv_rn(__fadd_rn(s.y, s.w), 2.f);
  const float w = __fsub_rn(s.z, s.x), h = __fsub_rn(s.w, s.y);
  return make_float4(__fsub_rn(xc, __fdiv_rn(w, 2.f)), __fsub_rn(yc, __fdiv_rn(h, 2.f)), w, h);
}

}  // namespace yv6
