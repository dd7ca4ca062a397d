// yv6_lite.cu -- the layers of the YOLOv6Lite networks that are not a dense convolution (include/yv6.h, "YOLOv6Lite"):
//   * yv6_dwconv_fwd     : depthwise k x k conv (k = 3 | 5, stride 1 | 2) + folded BN / bias + optional Hardswish
//                          (ConvBN / ConvBNHS with groups = C, DPBlock.conv_dw_1; reference layers/common.py:783-934)
//   * yv6_se_fwd         : SEBlock (common.py:740-768): mean over H x W, relu(W1 m + b1), hardsigmoid(W2 h + b2), x *= s
//   * yv6_channel_shuffle: channel_shuffle(cat(a, b), 2) (common.py:771-780, 822-823): y[2j] = a[j], y[2j+1] = b[j]
//   * yv6_upsample2x     : nn.Upsample(scale_factor=2, mode='nearest') of Lite_EffiNeck (reppan.py:1147-1149)
// All of them are memory-bound.  Activations are NHWC bf16 channel slices (base pointer + channel pitch), one plane or the
// three bf16 planes (hi, mid, lo) of the fp32-equivalent mode; in that mode every value is read as the fp32 sum of its
// planes, computed in fp32 and written back as three planes (the split of ops.split3).  yv6_dwconv_fwd_f16 and yv6_se_fwd with
// reserved0 = YV6_DT_F16 run the same kernels on one plane of fp16 activations (T = __half below).
#include <type_traits>

#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace yv6 {
namespace {

__device__ __forceinline__ float hardswish(float v) { return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f); }   // nn.Hardswish
__device__ __forceinline__ float hardsigmoid(float v) { return fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f); }    // nn.Hardsigmoid

__device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_float(__half v) { return __half2float(v); }

template <typename T>
__device__ __forceinline__ float load_val(const T* p, int64_t plane_stride, int planes) {
  float v = to_float(p[0]);
  for (int pl = 1; pl < planes; ++pl) v += to_float(p[pl * plane_stride]);
  return v;
}

__device__ __forceinline__ void store_val(__half* p, int64_t, int, float v) { p[0] = __float2half_rn(v); }   // one plane
__device__ __forceinline__ void store_val(__nv_bfloat16* p, int64_t plane_stride, int planes, float v) {
  const __nv_bfloat16 hi = __float2bfloat16(v);
  p[0] = hi;
  if (planes == 3) {
    const float r1 = v - __bfloat162float(hi);
    const __nv_bfloat16 mid = __float2bfloat16(r1);
    p[plane_stride] = mid;
    p[2 * plane_stride] = __float2bfloat16(r1 - __bfloat162float(mid));
  }
}

// ------------------------------------------------------------------------------------------------
// depthwise conv: one CTA = an 8 x 16 output tile x 8 channels of one image, one thread = one output pixel x 8 channels.
// The input window of the tile (halo included, zero outside the image) is staged once in shared memory as fp32, so each
// input value is read from global memory once per CTA instead of k*k / s^2 times.  Channel vectors are 16-byte loads and
// stores where the slice allows it (pitch % 8 == 0, 16-byte aligned slice start, 8 channels left); a scalar path takes the
// rest, so any channel count and offset works and channels outside [0, C) are never written.
// ------------------------------------------------------------------------------------------------
constexpr int kDwTH = 8, kDwTW = 16, kDwCV = 8, kDwThreads = kDwTH * kDwTW;

struct DwParams {
  const void* x;            // bf16 or fp16 (T)
  const float* w;           // [k*k][C]
  const float* b;           // [C] or null
  void* y;
  int64_t x_pitch, y_pitch, x_plane, y_plane;
  int32_t N, H, W, C, Ho, Wo, act, planes, x_vec, y_vec, tiles_w;
};

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (std::is_same_v<T, __half>) {
    const __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  } else {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  }
}
template <typename T> struct Pair2;
template <> struct Pair2<__nv_bfloat16> { using type = __nv_bfloat162; };
template <> struct Pair2<__half> { using type = __half2; };

template <int K, int S, typename T>
__device__ __forceinline__ void dwconv_body(const DwParams& p) {
  constexpr int IH = (kDwTH - 1) * S + K, IW = (kDwTW - 1) * S + K;
  __shared__ float4 tile[IH * IW * 2];
  __shared__ float wsm[K * K * kDwCV];
  __shared__ float bsm[kDwCV];
  const int tid = threadIdx.x;
  const int n = blockIdx.z, c0 = blockIdx.y * kDwCV, nc = min(kDwCV, p.C - c0);
  const int ho0 = (blockIdx.x / p.tiles_w) * kDwTH, wo0 = (blockIdx.x % p.tiles_w) * kDwTW;
  const int hi0 = ho0 * S - K / 2, wi0 = wo0 * S - K / 2;
  for (int i = tid; i < K * K * kDwCV; i += kDwThreads) {
    const int c = i % kDwCV;
    wsm[i] = c < nc ? p.w[(int64_t)(i / kDwCV) * p.C + c0 + c] : 0.f;
  }
  if (tid < kDwCV) bsm[tid] = (p.b != nullptr && tid < nc) ? p.b[c0 + tid] : 0.f;
  const bool vec_x = p.x_vec && nc == kDwCV;
  for (int i = tid; i < IH * IW; i += kDwThreads) {
    const int h = hi0 + i / IW, w = wi0 + i % IW;
    float v[kDwCV];
#pragma unroll
    for (int c = 0; c < kDwCV; ++c) v[c] = 0.f;
    if (h >= 0 && h < p.H && w >= 0 && w < p.W) {
      const T* src = static_cast<const T*>(p.x) + ((int64_t)(n * p.H + h) * p.W + w) * p.x_pitch + c0;
      for (int pl = 0; pl < p.planes; ++pl, src += p.x_plane) {
        if (vec_x) {
          const uint4 q = __ldg(reinterpret_cast<const uint4*>(src));
          const uint32_t u[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const typename Pair2<T>::type b2 = *reinterpret_cast<const typename Pair2<T>::type*>(&u[j]);
            v[2 * j] += __low2float(b2);
            v[2 * j + 1] += __high2float(b2);
          }
        } else {
          for (int c = 0; c < nc; ++c) v[c] += to_float(src[c]);
        }
      }
    }
    tile[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
    tile[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
  }
  __syncthreads();
  const int ty = tid / kDwTW, tx = tid % kDwTW, ho = ho0 + ty, wo = wo0 + tx;
  if (ho >= p.Ho || wo >= p.Wo) return;
  float acc[kDwCV];
#pragma unroll
  for (int c = 0; c < kDwCV; ++c) acc[c] = bsm[c];
#pragma unroll
  for (int r = 0; r < K; ++r) {
#pragma unroll
    for (int q = 0; q < K; ++q) {
      const int i = (ty * S + r) * IW + tx * S + q;
      const float4 a = tile[2 * i], b = tile[2 * i + 1];
      const float* wt = wsm + (r * K + q) * kDwCV;
      acc[0] = fmaf(a.x, wt[0], acc[0]); acc[1] = fmaf(a.y, wt[1], acc[1]);
      acc[2] = fmaf(a.z, wt[2], acc[2]); acc[3] = fmaf(a.w, wt[3], acc[3]);
      acc[4] = fmaf(b.x, wt[4], acc[4]); acc[5] = fmaf(b.y, wt[5], acc[5]);
      acc[6] = fmaf(b.z, wt[6], acc[6]); acc[7] = fmaf(b.w, wt[7], acc[7]);
    }
  }
  if (p.act == YV6_ACT_HARDSWISH) {
#pragma unroll
    for (int c = 0; c < kDwCV; ++c) acc[c] = hardswish(acc[c]);
  }
  T* dst = static_cast<T*>(p.y) + ((int64_t)(n * p.Ho + ho) * p.Wo + wo) * p.y_pitch + c0;
  if (p.planes == 1 && p.y_vec && nc == kDwCV) {
    uint4 q;
    uint32_t* u = reinterpret_cast<uint32_t*>(&q);
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = pack2<T>(acc[2 * j], acc[2 * j + 1]);
    *reinterpret_cast<uint4*>(dst) = q;
  } else {
#pragma unroll
    for (int c = 0; c < kDwCV; ++c)
      if (c < nc) store_val(dst + c, p.y_plane, p.planes, acc[c]);
  }
}

template <int K, int S>
__global__ void __launch_bounds__(kDwThreads) dwconv_kernel(const DwParams p) { dwconv_body<K, S, __nv_bfloat16>(p); }
template <int K, int S>
__global__ void __launch_bounds__(kDwThreads) dwconv_f16_kernel(const DwParams p) { dwconv_body<K, S, __half>(p); }

// ------------------------------------------------------------------------------------------------
// squeeze-excite: one CTA per image does the whole block -- the mean, both FCs and the scaling -- so nothing crosses CTAs:
// every sum has a fixed order (thread (phase, c) adds pixels phase, phase + P, ... in float64; the phases are added in
// order) and two runs give bit-identical results.  The scaling pass re-reads the slice, mostly from L2.
// ------------------------------------------------------------------------------------------------
constexpr int kSeThreads = 512, kSeMaxC = 512, kSeMaxCr = 128;

struct SeParams {
  void* x;                  // bf16 or fp16 (T)
  const float *w1, *b1, *w2, *b2;
  int64_t pitch, plane;
  int32_t HW, C, Cr, planes;
};

template <typename T>
__device__ __forceinline__ void se_body(const SeParams& p) {
  __shared__ double part[kSeThreads];
  __shared__ float mean[kSeMaxC], hid[kSeMaxCr], scale[kSeMaxC];
  const int t = threadIdx.x, C = p.C, P = kSeThreads / C;
  T* x = static_cast<T*>(p.x) + (int64_t)blockIdx.x * p.HW * p.pitch;
  const int c = t % C, ph = t / C;
  if (ph < P) {
    double s = 0.0;
    for (int i = ph; i < p.HW; i += P) s += (double)load_val(x + (int64_t)i * p.pitch + c, p.plane, p.planes);
    part[t] = s;
  }
  __syncthreads();
  if (t < C) {
    double s = 0.0;
    for (int j = 0; j < P; ++j) s += part[j * C + t];
    mean[t] = (float)(s / p.HW);
  }
  __syncthreads();
  if (t < p.Cr) {
    float h = p.b1[t];
    for (int j = 0; j < C; ++j) h = fmaf(p.w1[(int64_t)t * C + j], mean[j], h);
    hid[t] = fmaxf(h, 0.f);
  }
  __syncthreads();
  if (t < C) {
    float z = p.b2[t];
    for (int j = 0; j < p.Cr; ++j) z = fmaf(p.w2[(int64_t)t * p.Cr + j], hid[j], z);
    scale[t] = hardsigmoid(z);
  }
  __syncthreads();
  for (int64_t i = t; i < (int64_t)p.HW * C; i += kSeThreads) {
    T* e = x + (i / C) * p.pitch + i % C;
    store_val(e, p.plane, p.planes, load_val(e, p.plane, p.planes) * scale[i % C]);
  }
}

__global__ void __launch_bounds__(kSeThreads) se_kernel(const SeParams p) { se_body<__nv_bfloat16>(p); }
__global__ void __launch_bounds__(kSeThreads) se_f16_kernel(const SeParams p) { se_body<__half>(p); }

// ------------------------------------------------------------------------------------------------
// channel shuffle / nearest 2x upsample: one thread per output element (and plane).  These move a few hundred KB per
// image; the plane values are copied bit for bit.
// ------------------------------------------------------------------------------------------------
struct CopyParams {
  const __nv_bfloat16 *a, *b;
  __nv_bfloat16* y;
  int64_t a_pitch, b_pitch, y_pitch, a_plane, b_plane, y_plane;
  int64_t total;            // output elements per plane
  int32_t C, H, W, planes;  // shuffle: C per source; upsample: C channels of an H x W source
};

__global__ void shuffle_kernel(const CopyParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.total) return;
  const int64_t pix = i / (2 * p.C);
  const int oc = (int)(i % (2 * p.C)), c = oc >> 1;
  const __nv_bfloat16* s = (oc & 1) ? p.b + pix * p.b_pitch + c : p.a + pix * p.a_pitch + c;
  const int64_t sp = (oc & 1) ? p.b_plane : p.a_plane;
  __nv_bfloat16* d = p.y + pix * p.y_pitch + oc;
  for (int pl = 0; pl < p.planes; ++pl) d[pl * p.y_plane] = s[pl * sp];
}

__global__ void upsample2x_kernel(const CopyParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.total) return;
  const int c = (int)(i % p.C);
  const int64_t opix = i / p.C;                       // (n, oh, ow) of the 2H x 2W output
  const int ow = (int)(opix % (2 * p.W));
  const int64_t r = opix / (2 * p.W);
  const int oh = (int)(r % (2 * p.H));
  const int64_t n = r / (2 * p.H);
  const __nv_bfloat16* s = p.a + ((n * p.H + oh / 2) * p.W + ow / 2) * p.a_pitch + c;
  __nv_bfloat16* d = p.y + opix * p.y_pitch + c;
  for (int pl = 0; pl < p.planes; ++pl) d[pl * p.y_plane] = s[pl * p.a_plane];
}

template <int K, int S>
cudaError_t launch_dw(const DwParams& p, dim3 grid, cudaStream_t st, bool f16) {
  if (f16) dwconv_f16_kernel<K, S><<<grid, kDwThreads, 0, st>>>(p);
  else dwconv_kernel<K, S><<<grid, kDwThreads, 0, st>>>(p);
  return cudaGetLastError();
}

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

}  // namespace
}  // namespace yv6

using namespace yv6;

static int dwconv_fwd(yv6_handle* h, const yv6_dw_desc* d, void* stream, bool f16) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->x && d->w && d->y, "dwconv: null argument");
  YV6_REQUIRE(!f16 || d->nsplit == 1, "dwconv_f16: nsplit must be 1");
  YV6_REQUIRE((d->k == 3 || d->k == 5) && (d->stride == 1 || d->stride == 2), "dwconv: k=%d stride=%d (k in {3,5}, stride in {1,2})",
              d->k, d->stride);
  YV6_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->N <= 65535, "dwconv: bad shape %dx%dx%dx%d", d->N, d->H, d->W, d->C);
  YV6_REQUIRE(d->x_c_total >= d->C && d->y_c_total >= d->C, "dwconv: pitch below C");
  YV6_REQUIRE(d->act == YV6_ACT_NONE || d->act == YV6_ACT_HARDSWISH, "dwconv: act %d (none or hardswish)", d->act);
  YV6_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "dwconv: nsplit %d", d->nsplit);
  DwParams p;
  p.x = d->x;
  p.w = d->w;
  p.b = d->bias;
  p.y = d->y;
  p.x_pitch = d->x_c_total, p.y_pitch = d->y_c_total, p.x_plane = d->x_plane_stride, p.y_plane = d->y_plane_stride;
  p.N = d->N, p.H = d->H, p.W = d->W, p.C = d->C;
  p.Ho = (d->H - 1) / d->stride + 1, p.Wo = (d->W - 1) / d->stride + 1;   // padding k / 2
  p.act = d->act, p.planes = d->nsplit;
  p.x_vec = d->x_c_total % 8 == 0 && aligned16(d->x) && (d->nsplit == 1 || d->x_plane_stride % 8 == 0);
  p.y_vec = d->y_c_total % 8 == 0 && aligned16(d->y);
  p.tiles_w = (p.Wo + kDwTW - 1) / kDwTW;
  const dim3 grid(p.tiles_w * ((p.Ho + kDwTH - 1) / kDwTH), (d->C + kDwCV - 1) / kDwCV, d->N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (d->k == 3) e = d->stride == 1 ? launch_dw<3, 1>(p, grid, st, f16) : launch_dw<3, 2>(p, grid, st, f16);
  else e = d->stride == 1 ? launch_dw<5, 1>(p, grid, st, f16) : launch_dw<5, 2>(p, grid, st, f16);
  YV6_CHECK_CUDA(e);
  return YV6_OK;
}

extern "C" int yv6_dwconv_fwd(yv6_handle* h, const yv6_dw_desc* d, void* stream) { return dwconv_fwd(h, d, stream, false); }
extern "C" int yv6_dwconv_fwd_f16(yv6_handle* h, const yv6_dw_desc* d, void* stream) { return dwconv_fwd(h, d, stream, true); }

extern "C" int yv6_se_fwd(yv6_handle* h, const yv6_se_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->x && d->w1 && d->b1 && d->w2 && d->b2, "se: null argument");
  YV6_REQUIRE(d->C > 0 && d->C <= kSeMaxC && d->Cr > 0 && d->Cr <= kSeMaxCr, "se: C=%d Cr=%d (C <= %d, Cr <= %d)", d->C, d->Cr,
              kSeMaxC, kSeMaxCr);
  YV6_REQUIRE(d->N > 0 && d->HW > 0 && d->c_total >= d->C, "se: bad shape N=%d HW=%d", d->N, d->HW);
  YV6_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "se: nsplit %d", d->nsplit);
  YV6_REQUIRE(d->reserved0 == 0 || (d->reserved0 == YV6_DT_F16 && d->nsplit == 1), "se: operand dtype %d (0 = bf16, or YV6_DT_F16 with nsplit 1)",
              d->reserved0);
  SeParams p{d->x, d->w1, d->b1, d->w2, d->b2, d->c_total, d->plane_stride, d->HW, d->C, d->Cr, d->nsplit};
  if (d->reserved0 == YV6_DT_F16) se_f16_kernel<<<d->N, kSeThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  else se_kernel<<<d->N, kSeThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_channel_shuffle(yv6_handle* h, const void* a, int64_t a_pitch, int64_t a_plane, const void* b, int64_t b_pitch,
                                   int64_t b_plane, int64_t pixels, int32_t C, void* y, int64_t y_pitch, int64_t y_plane,
                                   int32_t nsplit, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && a && b && y, "channel_shuffle: null argument");
  YV6_REQUIRE(C > 0 && pixels > 0 && a_pitch >= C && b_pitch >= C && y_pitch >= 2 * C, "channel_shuffle: bad shape");
  YV6_REQUIRE(nsplit == 1 || nsplit == 3, "channel_shuffle: nsplit %d", nsplit);
  CopyParams p{static_cast<const __nv_bfloat16*>(a), static_cast<const __nv_bfloat16*>(b), static_cast<__nv_bfloat16*>(y),
               a_pitch, b_pitch, y_pitch, a_plane, b_plane, y_plane, pixels * 2 * C, C, 0, 0, nsplit};
  shuffle_kernel<<<(unsigned)((p.total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_upsample2x(yv6_handle* h, const void* x, int64_t x_pitch, int64_t x_plane, int32_t N, int32_t H, int32_t W,
                              int32_t C, void* y, int64_t y_pitch, int64_t y_plane, int32_t nsplit, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && x && y, "upsample2x: null argument");
  YV6_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && x_pitch >= C && y_pitch >= C, "upsample2x: bad shape");
  YV6_REQUIRE(nsplit == 1 || nsplit == 3, "upsample2x: nsplit %d", nsplit);
  CopyParams p{static_cast<const __nv_bfloat16*>(x), nullptr, static_cast<__nv_bfloat16*>(y), x_pitch, 0, y_pitch, x_plane, 0, y_plane,
               (int64_t)N * 4 * H * W * C, C, H, W, nsplit};
  upsample2x_kernel<<<(unsigned)((p.total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
