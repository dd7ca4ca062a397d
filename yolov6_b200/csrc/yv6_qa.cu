// yv6_qa.cu -- the training kernels of QARepVGGBlock / QARepVGGBlockV2 (include/yv6.h, "QARepVGGBlock"; reference
// layers/common.py:322-477).  Their BatchNorm sits AFTER the branch sum, so the multi-branch BN kernels of yv6_train.cu
// (one BN per branch, summed after normalisation) cannot express the block.  The training engine runs
//   u = conv3x3(x), v = conv1x1(x)                  yv6_conv_fwd (raw)
//   BN_d statistics of u                            yv6_bn_stats_finalize (nb = 1)
//   t = BN_d(u) + v [+ x [+ avg3x3(x)]], BN_p stats yv6_qa_fwd (this file, one launch)
//   y = relu(BN_p(t)) [+ alpha * res]               yv6_bn_apply_fwd (nb = 1)
// and in the backward pass yv6_bn_bwd twice (BN_p, then BN_d with dy = dt) plus yv6_qa_bwd for the parameter-free identity
// and average-pool branches: g(x) (+)= dt + avg3x3^T(dt).
//
// Both kernels are memory-bound.  One CTA = an 8 x 16 pixel tile x 8 channels, looping over images; one thread = one pixel
// x 8 channels.  The 3x3 neighbourhood (x forward, dt backward) is staged once per tile in shared memory as fp32, as
// yv6_lite.cu's dwconv_kernel does.  Channel vectors are 16-byte loads / stores where the slice allows them (pitch % 8 == 0,
// 16-byte aligned start, 8 channels left); a scalar path takes the rest, so any C and channel offset works.
#include <algorithm>
#include <cstring>

#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace yv6 {
namespace {

constexpr int kQaTH = 8, kQaTW = 16, kQaCV = 8, kQaThreads = kQaTH * kQaTW;
constexpr int kQaIH = kQaTH + 2, kQaIW = kQaTW + 2;

bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

__device__ __forceinline__ void load8(const __nv_bfloat16* p, bool vec, int nc, float (&v)[kQaCV]) {
  if (vec) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 b2 = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
      v[2 * j] = __low2float(b2);
      v[2 * j + 1] = __high2float(b2);
    }
  } else {
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) v[c] = c < nc ? __bfloat162float(p[c]) : 0.f;
  }
}

// rounds v to bf16 in place (the stored value) and writes it
__device__ __forceinline__ void store8(__nv_bfloat16* p, bool vec, int nc, float (&v)[kQaCV]) {
  if (vec) {
    uint4 q;
    uint32_t* w = reinterpret_cast<uint32_t*>(&q);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 b2 = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
      w[j] = *reinterpret_cast<const uint32_t*>(&b2);
      v[2 * j] = __low2float(b2);
      v[2 * j + 1] = __high2float(b2);
    }
    *reinterpret_cast<uint4*>(p) = q;
  } else {
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) {
      const __nv_bfloat16 b = __float2bfloat16(v[c]);
      v[c] = __bfloat162float(b);
      if (c < nc) p[c] = b;
    }
  }
}

// the (kQaTH + 2) x (kQaTW + 2) window around a tile, zero outside the image, as fp32 [pixel][8 channels]
__device__ __forceinline__ void stage_window(float4* win, const __nv_bfloat16* src, int64_t pitch, bool vec, int nc, int n, int H,
                                             int W, int h0, int w0) {
  for (int i = threadIdx.x; i < kQaIH * kQaIW; i += kQaThreads) {
    const int h = h0 - 1 + i / kQaIW, w = w0 - 1 + i % kQaIW;
    float v[kQaCV];
    if (h >= 0 && h < H && w >= 0 && w < W) {
      load8(src + ((int64_t)(n * H + h) * W + w) * pitch, vec, nc, v);
    } else {
#pragma unroll
      for (int c = 0; c < kQaCV; ++c) v[c] = 0.f;
    }
    win[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
    win[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// centre (ty, tx) of the staged window, and (with_box) the 3x3 box sum around it
__device__ __forceinline__ void window_at(const float4* win, int ty, int tx, bool with_box, float (&ctr)[kQaCV], float (&box)[kQaCV]) {
  const int ic = (ty + 1) * kQaIW + tx + 1;
  const float4 a = win[2 * ic], b = win[2 * ic + 1];
  ctr[0] = a.x; ctr[1] = a.y; ctr[2] = a.z; ctr[3] = a.w; ctr[4] = b.x; ctr[5] = b.y; ctr[6] = b.z; ctr[7] = b.w;
#pragma unroll
  for (int c = 0; c < kQaCV; ++c) box[c] = 0.f;
  if (!with_box) return;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const int i = (ty + r) * kQaIW + tx + q;
      const float4 e = win[2 * i], f = win[2 * i + 1];
      box[0] += e.x; box[1] += e.y; box[2] += e.z; box[3] += e.w;
      box[4] += f.x; box[5] += f.y; box[6] += f.z; box[7] += f.w;
    }
  }
}

struct QaParams {
  const __nv_bfloat16 *u, *v, *x, *dt;
  __nv_bfloat16 *t, *dx;
  int64_t u_pitch, v_pitch, x_pitch, t_pitch, dt_pitch, dx_pitch;
  const float *scale_d, *shift_d, *gamma, *beta;
  float *rmean, *rvar, *stats;
  double* sums;
  unsigned int* counter;
  float eps, momentum;
  int32_t N, H, W, C, avg, accumulate, tiles_w;
  int32_t u_vec, v_vec, x_vec, t_vec, dt_vec, dx_vec;
};

// nn.BatchNorm2d in training mode from the float64 sums (as yv6_train.cu's bn_finalize_one): mean, biased variance for the
// normalisation, unbiased variance for the running statistics
__device__ __forceinline__ void finalize_channel(const QaParams& p, int c) {
  const double count = (double)p.N * p.H * p.W;
  const double m = __ldcg(p.sums + c) / count;
  double var = __ldcg(p.sums + p.C + c) / count - m * m;
  if (var < 0) var = 0;
  const double inv = 1.0 / sqrt(var + (double)p.eps);
  const double g = p.gamma[c];
  p.stats[c] = (float)m;
  p.stats[p.C + c] = (float)inv;
  p.stats[2 * p.C + c] = (float)(g * inv);
  p.stats[3 * p.C + c] = (float)((double)p.beta[c] - m * g * inv);
  if (p.rmean != nullptr) {
    const double unb = count > 1 ? var * count / (count - 1.0) : var;
    p.rmean[c] = (float)((1.0 - p.momentum) * p.rmean[c] + p.momentum * m);
    p.rvar[c] = (float)((1.0 - p.momentum) * p.rvar[c] + p.momentum * unb);
  }
}

template <bool HAS_X>
__global__ void __launch_bounds__(kQaThreads) qa_fwd_kernel(const QaParams p) {
  __shared__ float4 win[HAS_X ? kQaIH * kQaIW * 2 : 1];
  __shared__ float red[2][kQaThreads / 32][kQaCV];
  __shared__ int s_last;
  const int tid = threadIdx.x, c0 = blockIdx.y * kQaCV, nc = min(kQaCV, p.C - c0);
  const int h0 = (blockIdx.x / p.tiles_w) * kQaTH, w0 = (blockIdx.x % p.tiles_w) * kQaTW;
  const int ty = tid / kQaTW, tx = tid % kQaTW, h = h0 + ty, w = w0 + tx;
  const bool inside = h < p.H && w < p.W;
  const bool full = nc == kQaCV;
  float sc[kQaCV], sh[kQaCV], s[kQaCV], q[kQaCV];
#pragma unroll
  for (int c = 0; c < kQaCV; ++c) {
    sc[c] = c < nc ? __ldg(p.scale_d + c0 + c) : 0.f;
    sh[c] = c < nc ? __ldg(p.shift_d + c0 + c) : 0.f;
    s[c] = q[c] = 0.f;
  }
  for (int n = blockIdx.z; n < p.N; n += gridDim.z) {
    float ctr[kQaCV], box[kQaCV];
    if (HAS_X) {
      __syncthreads();                          // the previous image's window is no longer read
      stage_window(win, p.x + c0, p.x_pitch, p.x_vec && full, nc, n, p.H, p.W, h0, w0);
      __syncthreads();
      window_at(win, ty, tx, p.avg != 0, ctr, box);
    }
    if (!inside) continue;
    const int64_t px = (int64_t)(n * p.H + h) * p.W + w;
    float a[kQaCV], b[kQaCV];
    load8(p.u + px * p.u_pitch + c0, p.u_vec && full, nc, a);
    load8(p.v + px * p.v_pitch + c0, p.v_vec && full, nc, b);
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) {
      float t = fmaf(a[c], sc[c], sh[c]) + b[c];
      if (HAS_X) t = t + ctr[c] + box[c] * (1.f / 9.f);      // box is zero without the avg branch
      a[c] = t;
    }
    store8(p.t + px * p.t_pitch + c0, p.t_vec && full, nc, a);
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) {                       // statistics of the stored (rounded) values
      s[c] += a[c];
      q[c] = fmaf(a[c], a[c], q[c]);
    }
  }
  // warp sums, then one float64 atomic per channel and CTA
#pragma unroll
  for (int c = 0; c < kQaCV; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
      q[c] += __shfl_xor_sync(0xffffffffu, q[c], o);
    }
  }
  if ((tid & 31) == 0) {
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) {
      red[0][tid >> 5][c] = s[c];
      red[1][tid >> 5][c] = q[c];
    }
  }
  __syncthreads();
  if (tid < 2 * kQaCV) {
    const int which = tid / kQaCV, c = tid % kQaCV;
    if (c < nc) {
      double acc = 0.0;
#pragma unroll
      for (int wp = 0; wp < kQaThreads / 32; ++wp) acc += (double)red[which][wp][c];
      atomicAdd(p.sums + which * p.C + c0 + c, acc);
    }
  }
  // the CTA that finishes last finalises the post-sum BatchNorm
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int total = gridDim.x * gridDim.y * gridDim.z;
    s_last = atomicAdd(p.counter, 1u) == total - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int c = tid; c < p.C; c += kQaThreads) finalize_channel(p, c);
}

template <bool AVG>
__global__ void __launch_bounds__(kQaThreads) qa_bwd_kernel(const QaParams p) {
  __shared__ float4 win[AVG ? kQaIH * kQaIW * 2 : 1];
  const int tid = threadIdx.x, c0 = blockIdx.y * kQaCV, nc = min(kQaCV, p.C - c0);
  const int h0 = (blockIdx.x / p.tiles_w) * kQaTH, w0 = (blockIdx.x % p.tiles_w) * kQaTW;
  const int ty = tid / kQaTW, tx = tid % kQaTW, h = h0 + ty, w = w0 + tx;
  const bool inside = h < p.H && w < p.W;
  const bool full = nc == kQaCV;
  for (int n = blockIdx.z; n < p.N; n += gridDim.z) {
    float g[kQaCV], box[kQaCV];
    const int64_t px = (int64_t)(n * p.H + h) * p.W + w;
    if (AVG) {
      // AvgPool2d(3, 1, 1) with count_include_pad divides every window by 9, so its adjoint is the same box filter
      __syncthreads();
      stage_window(win, p.dt + c0, p.dt_pitch, p.dt_vec && full, nc, n, p.H, p.W, h0, w0);
      __syncthreads();
      window_at(win, ty, tx, true, g, box);
    } else if (inside) {
      load8(p.dt + px * p.dt_pitch + c0, p.dt_vec && full, nc, g);
    }
    if (!inside) continue;
    __nv_bfloat16* dst = p.dx + px * p.dx_pitch + c0;
    float prev[kQaCV];
    if (p.accumulate) load8(dst, p.dx_vec && full, nc, prev);
#pragma unroll
    for (int c = 0; c < kQaCV; ++c) {
      float v = g[c];
      if (AVG) v += box[c] * (1.f / 9.f);
      g[c] = p.accumulate ? prev[c] + v : v;
    }
    store8(dst, p.dx_vec && full, nc, g);
  }
}

void fill_params(yv6_handle* h, const yv6_qa_desc* d, QaParams* p, dim3* grid) {
  memset(p, 0, sizeof(*p));
  p->u = static_cast<const __nv_bfloat16*>(d->u), p->v = static_cast<const __nv_bfloat16*>(d->v);
  p->x = static_cast<const __nv_bfloat16*>(d->x), p->dt = static_cast<const __nv_bfloat16*>(d->dt);
  p->t = static_cast<__nv_bfloat16*>(d->t), p->dx = static_cast<__nv_bfloat16*>(d->dx);
  p->u_pitch = d->u_pitch, p->v_pitch = d->v_pitch, p->x_pitch = d->x_pitch, p->t_pitch = d->t_pitch;
  p->dt_pitch = d->dt_pitch, p->dx_pitch = d->dx_pitch;
  p->scale_d = d->scale_d, p->shift_d = d->shift_d, p->gamma = d->gamma, p->beta = d->beta;
  p->rmean = d->running_mean, p->rvar = d->running_var, p->stats = d->stats;
  p->sums = d->sums, p->counter = d->counter, p->eps = d->eps, p->momentum = d->momentum;
  p->N = d->N, p->H = d->H, p->W = d->W, p->C = d->C, p->avg = d->avg, p->accumulate = d->accumulate;
  auto vec = [](const void* ptr, int64_t pitch) { return (int32_t)(ptr != nullptr && pitch % 8 == 0 && aligned16(ptr)); };
  p->u_vec = vec(d->u, d->u_pitch), p->v_vec = vec(d->v, d->v_pitch), p->x_vec = vec(d->x, d->x_pitch);
  p->t_vec = vec(d->t, d->t_pitch), p->dt_vec = vec(d->dt, d->dt_pitch), p->dx_vec = vec(d->dx, d->dx_pitch);
  p->tiles_w = (d->W + kQaTW - 1) / kQaTW;
  const int tiles = p->tiles_w * ((d->H + kQaTH - 1) / kQaTH), cgs = (d->C + kQaCV - 1) / kQaCV;
  // enough CTAs to fill the GPU several times over; each loops over its share of the images (fewer float64 atomics)
  const int target = 8 * h->num_sms;
  const int nz = std::max(1, std::min(d->N, (target + tiles * cgs - 1) / (tiles * cgs)));
  *grid = dim3(tiles, cgs, nz);
}

}  // namespace
}  // namespace yv6

using namespace yv6;

extern "C" int yv6_qa_fwd(yv6_handle* h, const yv6_qa_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->u && d->v && d->scale_d && d->shift_d && d->t, "qa_fwd: null argument");
  YV6_REQUIRE(d->sums && d->counter && d->stats && d->gamma && d->beta, "qa_fwd: null statistics argument");
  YV6_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && (int64_t)d->C <= 65535 * kQaCV, "qa_fwd: bad shape %dx%dx%dx%d",
              d->N, d->H, d->W, d->C);
  YV6_REQUIRE(d->u_pitch >= d->C && d->v_pitch >= d->C && d->t_pitch >= d->C && (!d->x || d->x_pitch >= d->C), "qa_fwd: pitch below C");
  YV6_REQUIRE(!d->avg || d->x, "qa_fwd: the average-pool branch needs x");
  QaParams p;
  dim3 grid;
  fill_params(h, d, &p, &grid);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!d->zeroed) {
    YV6_CHECK_CUDA(cudaMemsetAsync(d->sums, 0, sizeof(double) * 2 * d->C, s));
    YV6_CHECK_CUDA(cudaMemsetAsync(d->counter, 0, sizeof(uint32_t), s));
  }
  if (d->x) qa_fwd_kernel<true><<<grid, kQaThreads, 0, s>>>(p);
  else qa_fwd_kernel<false><<<grid, kQaThreads, 0, s>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_qa_bwd(yv6_handle* h, const yv6_qa_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->dt && d->dx, "qa_bwd: null argument");
  YV6_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && (int64_t)d->C <= 65535 * kQaCV, "qa_bwd: bad shape %dx%dx%dx%d",
              d->N, d->H, d->W, d->C);
  YV6_REQUIRE(d->dt_pitch >= d->C && d->dx_pitch >= d->C, "qa_bwd: pitch below C");
  QaParams p;
  dim3 grid;
  fill_params(h, d, &p, &grid);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (d->avg) qa_bwd_kernel<true><<<grid, kQaThreads, 0, s>>>(p);
  else qa_bwd_kernel<false><<<grid, kQaThreads, 0, s>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
