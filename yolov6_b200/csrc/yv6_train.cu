// yv6_train.cu -- the HBM-bound training kernels around the conv / wgrad GEMMs (sm_90a, CUDA cores).
//
// The reference trains in *train form*: every ConvModule is conv -> BatchNorm(batch stats) -> act
// (yolov6/layers/common.py:26-49) and every RepVGGBlock is relu(BN(conv3x3) + BN(conv1x1) + BN(x))
// with three independent BatchNorms (common.py:245-255); autograd + cuDNN then run the backward.
// Here each block is: raw conv(s) on tensor cores (yv6_conv_fwd with no bias/act) and
//   yv6_bn_stats      per-channel sum / sum-of-squares of an NHWC bf16 tensor            (fwd)
//   yv6_bn_finalize   mean / invstd / running-stat update (momentum .03, eps 1e-3)        (fwd)
//   yv6_bn_apply_fwd  y = act(sum_b (x_b * scale_b + shift_b)) over up to 3 branches      (fwd)
//   yv6_bn_bwd_reduce per branch: sum(dz), sum(dz * xhat_b) with dz = dY * act'(.)         (bwd)
//   yv6_bn_bwd_apply  per branch: dx_b = scale_b * (dz - S1/M - xhat_b * S2_b/M)           (bwd)
// plus yv6_head_grad_prep (sigmoid backward + repack of the head gradients), yv6_maxpool5_bwd (SPPF)
// and yv6_stem_wgrad (the 3-channel first conv).  All activations are NHWC bf16 with a channel pitch
// (slices of concat buffers); statistics and parameter gradients are float64 / float32.
#include <algorithm>

#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace yv6 {

constexpr int kTrThreads = 256;

struct View {          // NHWC bf16 tensor slice
  const __nv_bfloat16* p;
  int64_t pitch;       // elements between consecutive pixels
};

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 q = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const __nv_bfloat162 b2 = *reinterpret_cast<const __nv_bfloat162*>(&w[j]);
    v[2 * j] = __low2float(b2);
    v[2 * j + 1] = __high2float(b2);
  }
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&v)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    __nv_bfloat162 b2 = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    w[j] = *reinterpret_cast<uint32_t*>(&b2);
  }
  *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
}

// ---------------------------------------------------------------------------------- bn_stats
// grid: (channel groups of 8 per block.x dimension folded into threads) -- thread = (pixel lane, channel group)
__global__ void __launch_bounds__(kTrThreads) bn_stats_kernel(View x, int64_t pixels, int C, double* sum, double* sumsq) {
  const int cgs = C / 8;
  const int cg = threadIdx.x % cgs;                      // requires cgs | blockDim (host picks block = cgs * rows)
  const int prow = threadIdx.x / cgs, prows = blockDim.x / cgs;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  for (int64_t px = (int64_t)blockIdx.x * prows + prow; px < pixels; px += (int64_t)gridDim.x * prows) {
    float v[8];
    ld8(x.p + px * x.pitch + cg * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j] += v[j]; q[j] += v[j] * v[j]; }
  }
  // block-level reduction in shared memory first: one global atomic per channel per block instead of one per
  // thread (the per-thread version serialised on C addresses and cost 56 % of a training step)
  extern __shared__ double sred[];                      // [2][C]
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sred[c] = 0.0;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    atomicAdd(&sred[cg * 8 + j], (double)s[j]);
    atomicAdd(&sred[C + cg * 8 + j], (double)q[j]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(&sum[c], sred[c]);
    atomicAdd(&sumsq[c], sred[C + c]);
  }
}

// mean, biased var -> invstd, scale/shift; running stats with unbiased var (torch BatchNorm2d semantics)
__global__ void bn_finalize_kernel(const double* sum, const double* sumsq, double count, const float* gamma, const float* beta,
                                   float eps, float momentum, float* running_mean, float* running_var, float* mean_out,
                                   float* invstd_out, float* scale, float* shift, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = sum[c] / count;
  double var = sumsq[c] / count - m * m;
  if (var < 0) var = 0;
  const double inv = 1.0 / sqrt(var + (double)eps);
  mean_out[c] = (float)m;
  invstd_out[c] = (float)inv;
  const double g = gamma[c];
  scale[c] = (float)(g * inv);
  shift[c] = (float)((double)beta[c] - m * g * inv);
  if (running_mean != nullptr) {
    const double unb = (count > 1) ? var * count / (count - 1.0) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * m);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unb);
  }
}

// ---------------------------------------------------------------------------------- thread mapping
// All per-channel kernels below use thread = (pixel row `prow`, channel group `cg` of 8 channels = one 16-byte
// load); a thread keeps its channel group for the whole kernel, so the per-channel constants live in registers
// and the pixel loop is nothing but 16-byte loads, FMAs and (for the elementwise kernels) 16-byte stores.
struct ChanMap {
  int cgs, cg, prow, prows;
  __device__ __forceinline__ explicit ChanMap(int C) {
    cgs = C >> 3;
    cg = threadIdx.x % cgs;
    prow = threadIdx.x / cgs;
    prows = blockDim.x / cgs;
  }
};
__device__ __forceinline__ void ldc8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// column sums of per-thread partials: red[prows][C] floats in shared memory -> one double atomic per channel
__device__ __forceinline__ void block_colsum(const ChanMap& m, int C, const float (&part)[8], float* red, double* dst) {
  float4* row = reinterpret_cast<float4*>(red + (size_t)m.prow * C + m.cg * 8);
  row[0] = make_float4(part[0], part[1], part[2], part[3]);
  row[1] = make_float4(part[4], part[5], part[6], part[7]);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double a = 0.0;
    for (int r = 0; r < m.prows; ++r) a += (double)red[(size_t)r * C + c];
    atomicAdd(&dst[c], a);
  }
  __syncthreads();
}
// true in exactly one block per launch: the one that finishes last (its reads see every other block's atomics)
__device__ __forceinline__ bool last_block_done(unsigned int* counter) {
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last) __threadfence();
  return s_last != 0;
}
__device__ __forceinline__ double ld_cg(const double* p) { return __ldcg(p); }

// ---------------------------------------------------------------------------------- fused statistics
// sum / sum of squares of up to three branch inputs in ONE pass per branch tensor, then -- in the block that
// finishes last -- mean / invstd / scale / shift and the running-statistics update of every branch
// (nn.BatchNorm2d training semantics, eps / momentum as set by initialize_weights, torch_utils.py:38-48).
struct StatsParams {
  View x[3];
  int nb, C;
  int64_t pixels;
  double* sums;                 // [nb][2][C], zero on entry
  unsigned int* counter;        // zero on entry
  const float* gamma[3];
  const float* beta[3];
  float* rmean[3];
  float* rvar[3];
  float* stats[3];              // out [4][C]: mean, invstd, scale, shift; null = no finalize for that branch
  float eps, momentum;
};
__device__ __forceinline__ void bn_finalize_one(double sum, double sumsq, double count, float gamma, float beta, float eps,
                                                float momentum, float* rmean, float* rvar, float* stats, int C, int c) {
  const double m = sum / count;
  double var = sumsq / count - m * m;
  if (var < 0) var = 0;
  const double inv = 1.0 / sqrt(var + (double)eps);
  const double g = gamma;
  stats[c] = (float)m;
  stats[C + c] = (float)inv;
  stats[2 * C + c] = (float)(g * inv);
  stats[3 * C + c] = (float)((double)beta - m * g * inv);
  if (rmean != nullptr) {
    const double unb = (count > 1) ? var * count / (count - 1.0) : var;
    rmean[c] = (float)((1.0 - momentum) * rmean[c] + momentum * m);
    rvar[c] = (float)((1.0 - momentum) * rvar[c] + momentum * unb);
  }
}
template <int NB>
__global__ void __launch_bounds__(kTrThreads) bn_stats_multi_kernel(const StatsParams p) {
  extern __shared__ float red[];            // [prows][C]
  const ChanMap m(p.C);
  float s[NB][8], q[NB][8];
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int j = 0; j < 8; ++j) s[b][j] = q[b][j] = 0.f;
  if (m.prow < m.prows) {
    const int64_t step = (int64_t)gridDim.x * m.prows;
    for (int64_t px = (int64_t)blockIdx.x * m.prows + m.prow; px < p.pixels; px += 2 * step) {
      const bool two = (px + step) < p.pixels;
      float v0[NB][8], v1[NB][8];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        ld8(p.x[b].p + px * p.x[b].pitch + m.cg * 8, v0[b]);
        if (two) ld8(p.x[b].p + (px + step) * p.x[b].pitch + m.cg * 8, v1[b]);
      }
#pragma unroll
      for (int b = 0; b < NB; ++b) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[b][j] += v0[b][j]; q[b][j] += v0[b][j] * v0[b][j]; }
        if (two) {
#pragma unroll
          for (int j = 0; j < 8; ++j) { s[b][j] += v1[b][j]; q[b][j] += v1[b][j] * v1[b][j]; }
        }
      }
    }
  }
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    block_colsum(m, p.C, s[b], red, p.sums + (size_t)(2 * b) * p.C);
    block_colsum(m, p.C, q[b], red, p.sums + (size_t)(2 * b + 1) * p.C);
  }
  if (!last_block_done(p.counter)) return;
  for (int i = threadIdx.x; i < NB * p.C; i += blockDim.x) {
    const int b = i / p.C, c = i - b * p.C;
    if (p.stats[b] == nullptr) continue;
    bn_finalize_one(ld_cg(p.sums + (size_t)(2 * b) * p.C + c), ld_cg(p.sums + (size_t)(2 * b + 1) * p.C + c), (double)p.pixels,
                    p.gamma[b][c], p.beta[b][c], p.eps, p.momentum, p.rmean[b], p.rvar[b], p.stats[b], p.C, c);
  }
}

// ---------------------------------------------------------------------------------- bn_apply_fwd
struct ApplyParams {
  View x[3];
  const float* scale[3];
  const float* shift[3];
  int nb, act, C;
  int64_t pixels;
  __nv_bfloat16* y;
  int64_t y_pitch;
  View res;                  // optional shortcut: y = act(z) + alpha * res (BottleRep, common.py:600-617)
  float alpha;
  const float* alpha_dev;    // when set, the shortcut weight is read from device memory (no host sync, graph-capturable)
};
__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == YV6_ACT_RELU) return fmaxf(z, 0.f);
  if (act == YV6_ACT_SILU) return z / (1.f + __expf(-z));
  return z;
}
template <int NB>
__global__ void __launch_bounds__(kTrThreads) bn_apply_fwd_kernel(const ApplyParams p) {
  const ChanMap m(p.C);
  if (m.prow >= m.prows) return;
  float sc[NB][8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sh[j] = 0.f;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float t[8];
    ldc8(p.scale[b] + m.cg * 8, sc[b]);
    ldc8(p.shift[b] + m.cg * 8, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[j] += t[j];
  }
  const float alpha = (p.alpha_dev != nullptr) ? __ldg(p.alpha_dev) : p.alpha;
  const int64_t step = (int64_t)gridDim.x * m.prows;
  for (int64_t px = (int64_t)blockIdx.x * m.prows + m.prow; px < p.pixels; px += step) {
    float v[NB][8], r[8];
#pragma unroll
    for (int b = 0; b < NB; ++b) ld8(p.x[b].p + px * p.x[b].pitch + m.cg * 8, v[b]);
    if (p.res.p != nullptr) ld8(p.res.p + px * p.res.pitch + m.cg * 8, r);
    float z[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = sh[j];
#pragma unroll
      for (int b = 0; b < NB; ++b) a += v[b][j] * sc[b][j];
      z[j] = act_fwd(a, p.act);
    }
    if (p.res.p != nullptr) {
#pragma unroll
      for (int j = 0; j < 8; ++j) z[j] += alpha * r[j];
    }
    st8(p.y + px * p.y_pitch + m.cg * 8, z);
  }
}

// ---------------------------------------------------------------------------------- bn backward
struct BwdParams {
  View x[3];                 // branch inputs to their BN (raw conv outputs / block input for the identity branch)
  const float* mean[3];
  const float* invstd[3];
  const float* scale[3];     // gamma * invstd
  const float* shift[3];
  View dy;                   // gradient w.r.t. the block output
  View res;                  // optional shortcut input (y = act(z) + alpha * res)
  float alpha;
  const float* alpha_dev;
  __nv_bfloat16* dres;       // g(res) += alpha * dy  (= when dres_assign)
  int64_t dres_pitch;
  int dres_assign;
  double* dalpha;            // += sum dy * res
  int nb, act, C;
  int64_t pixels;
  double* s1;                // [C]      sum dz            (shared by the branches) = dbeta
  double* s2[3];             // [C] each sum dz * xhat_b   = dgamma_b (written by the last block of the reduce pass)
  double* work;              // [nb][C]  sum dz * x_b, zero on entry
  unsigned int* counter;     // zero on entry
  float* coef;               // [nb][2][C]: dx_b = scale_b * dz + coef[b][0] * x_b + coef[b][1]
  __nv_bfloat16* dx[3];
  int64_t dx_pitch[3];
  int accumulate[3];         // dx_b += ... instead of =
  double inv_count;
};
__device__ __forceinline__ void act_bwd(float (&dz)[8], const float (&z)[8], int act) {
  if (act == YV6_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 8; ++j) dz[j] = (z[j] > 0.f) ? dz[j] : 0.f;
  } else if (act == YV6_ACT_SILU) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-z[j]));
      dz[j] *= sg * (1.f + z[j] * (1.f - sg));
    }
  }
}
// pass 1: S1 = sum dz, T_b = sum dz * x_b (and dalpha); the last block turns them into dgamma_b and the
// coefficients of pass 2:  dx_b = scale_b (dz - S1/M - xhat_b S2_b/M) = scale_b dz + B_b x_b + C_b  with
// S2_b = invstd_b (T_b - mean_b S1), B_b = -scale_b invstd_b S2_b / M, C_b = -scale_b S1 / M - B_b mean_b.
template <int NB>
__global__ void __launch_bounds__(kTrThreads, 2) bn_bwd_reduce_kernel(const BwdParams p) {
  extern __shared__ float red[];            // [prows][C]
  const ChanMap m(p.C);
  float sc[NB][8], sh[8], a1[8], t[NB][8];
  float da = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { sh[j] = 0.f; a1[j] = 0.f; }
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float tmp[8];
    ldc8(p.scale[b] + m.cg * 8, sc[b]);
    ldc8(p.shift[b] + m.cg * 8, tmp);
#pragma unroll
    for (int j = 0; j < 8; ++j) { sh[j] += tmp[j]; t[b][j] = 0.f; }
  }
  if (m.prow < m.prows) {
    const int64_t step = (int64_t)gridDim.x * m.prows;
    for (int64_t px = (int64_t)blockIdx.x * m.prows + m.prow; px < p.pixels; px += step) {
      float dz[8], v[NB][8], z[8];
      ld8(p.dy.p + px * p.dy.pitch + m.cg * 8, dz);
#pragma unroll
      for (int b = 0; b < NB; ++b) ld8(p.x[b].p + px * p.x[b].pitch + m.cg * 8, v[b]);
      if (p.dalpha != nullptr) {
        float r[8];
        ld8(p.res.p + px * p.res.pitch + m.cg * 8, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) da += dz[j] * r[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float a = sh[j];
#pragma unroll
        for (int b = 0; b < NB; ++b) a += v[b][j] * sc[b][j];
        z[j] = a;
      }
      act_bwd(dz, z, p.act);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a1[j] += dz[j];
#pragma unroll
        for (int b = 0; b < NB; ++b) t[b][j] += dz[j] * v[b][j];
      }
    }
  }
  block_colsum(m, p.C, a1, red, p.s1);
#pragma unroll
  for (int b = 0; b < NB; ++b) block_colsum(m, p.C, t[b], red, p.work + (size_t)b * p.C);
  if (p.dalpha != nullptr) {
    // the block is cgs * rows threads, not always whole warps (C = 384: 240 threads, the last warp has 16 lanes): shuffle
    // among the lanes that exist only.  Lane 0 adds the same pairs in the same order as a full-warp xor butterfly would.
    const int lane = threadIdx.x & 31;
    const int lanes = min(32, (int)blockDim.x - (int)(threadIdx.x & ~31u));
    const unsigned mask = (lanes == 32) ? 0xffffffffu : ((1u << lanes) - 1u);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float other = __shfl_down_sync(mask, da, o);
      if (lane + o < lanes) da += other;
    }
    if (lane == 0) atomicAdd(p.dalpha, (double)da);
  }
  if (!last_block_done(p.counter)) return;
  for (int i = threadIdx.x; i < NB * p.C; i += blockDim.x) {
    const int b = i / p.C, c = i - b * p.C;
    const double S1 = ld_cg(p.s1 + c), T = ld_cg(p.work + (size_t)b * p.C + c);
    const double mean = p.mean[b][c], inv = p.invstd[b][c], scale = p.scale[b][c];
    const double S2 = inv * (T - mean * S1);
    p.s2[b][c] = S2;
    const double B = -scale * inv * S2 * p.inv_count;
    p.coef[(size_t)(2 * b) * p.C + c] = (float)B;
    p.coef[(size_t)(2 * b + 1) * p.C + c] = (float)(-scale * S1 * p.inv_count - B * mean);
  }
}

template <int NB>
__global__ void __launch_bounds__(kTrThreads, 2) bn_bwd_apply_kernel(const BwdParams p) {
  const ChanMap m(p.C);
  if (m.prow >= m.prows) return;
  float sc[NB][8], sh[8], cb[NB][8], cc[NB][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sh[j] = 0.f;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float tmp[8];
    ldc8(p.scale[b] + m.cg * 8, sc[b]);
    ldc8(p.shift[b] + m.cg * 8, tmp);
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[j] += tmp[j];
    ldc8(p.coef + (size_t)(2 * b) * p.C + m.cg * 8, cb[b]);
    ldc8(p.coef + (size_t)(2 * b + 1) * p.C + m.cg * 8, cc[b]);
  }
  const float alpha = (p.alpha_dev != nullptr) ? __ldg(p.alpha_dev) : p.alpha;
  const int64_t step = (int64_t)gridDim.x * m.prows;
  for (int64_t px = (int64_t)blockIdx.x * m.prows + m.prow; px < p.pixels; px += step) {
    float dz[8], v[NB][8], z[8];
    ld8(p.dy.p + px * p.dy.pitch + m.cg * 8, dz);
#pragma unroll
    for (int b = 0; b < NB; ++b) ld8(p.x[b].p + px * p.x[b].pitch + m.cg * 8, v[b]);
    if (p.dres != nullptr) {
      float old[8];
      __nv_bfloat16* dst = p.dres + px * p.dres_pitch + m.cg * 8;
      if (p.dres_assign) {
#pragma unroll
        for (int j = 0; j < 8; ++j) old[j] = alpha * dz[j];
      } else {
        ld8(dst, old);
#pragma unroll
        for (int j = 0; j < 8; ++j) old[j] += alpha * dz[j];
      }
      st8(dst, old);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = sh[j];
#pragma unroll
      for (int b = 0; b < NB; ++b) a += v[b][j] * sc[b][j];
      z[j] = a;
    }
    act_bwd(dz, z, p.act);
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = sc[b][j] * dz[j] + cb[b][j] * v[b][j] + cc[b][j];
      __nv_bfloat16* dst = p.dx[b] + px * p.dx_pitch[b] + m.cg * 8;
      if (p.accumulate[b]) {
        float old[8];
        ld8(dst, old);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += old[j];
      }
      st8(dst, o);
    }
  }
}

// ---------------------------------------------------------------------------------- head grad prep
// dlogit = dscore * s * (1 - s) (sigmoid backward, effidehead.py:85) or dreg; repacks level `l` of the
// [B, A, ch] fp32 head tensors into a dense NHWC bf16 tensor [B, H_l, W_l, ch_pad] (zero padded channels).
__global__ void __launch_bounds__(kTrThreads) head_grad_prep_kernel(const float* grad, const float* scores, int B, int A, int ch,
                                                                   int off, int hw, int ch_pad, __nv_bfloat16* out) {
  const int64_t total = (int64_t)B * hw * ch_pad;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % ch_pad);
    const int64_t px = i / ch_pad;
    const int b = (int)(px / hw), a = off + (int)(px % hw);
    float v = 0.f;
    if (c < ch) {
      const int64_t src = ((int64_t)b * A + a) * ch + c;
      v = grad[src];
      if (scores != nullptr) { const float s = scores[src]; v *= s * (1.f - s); }
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

// ---------------------------------------------------------------------------------- maxpool5 backward
// y = MaxPool2d(5, 1, 2)(x): scatter dy to the arg-max of each window (first maximum in row-major window
// order).  dx is fp32 [N,H,W,C] scratch (zeroed by the caller); x / dy are NHWC bf16 slices.
__global__ void __launch_bounds__(kTrThreads) maxpool5_bwd_kernel(View x, View dy, int N, int H, int W, int C, float* dx) {
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int w = (int)((i / C) % W), h = (int)((i / ((int64_t)C * W)) % H), n = (int)(i / ((int64_t)C * W * H));
    float best = -INFINITY;
    int bh = h, bw = w;
    for (int dyy = -2; dyy <= 2; ++dyy) {
      const int hh = h + dyy;
      if (hh < 0 || hh >= H) continue;
      for (int dxx = -2; dxx <= 2; ++dxx) {
        const int ww = w + dxx;
        if (ww < 0 || ww >= W) continue;
        const float v = __bfloat162float(x.p[(((int64_t)n * H + hh) * W + ww) * x.pitch + c]);
        if (v > best) { best = v; bh = hh; bw = ww; }
      }
    }
    const float g = __bfloat162float(dy.p[(((int64_t)n * H + h) * W + w) * dy.pitch + c]);
    atomicAdd(&dx[(((int64_t)n * H + bh) * W + bw) * C + c], g);
  }
}

// dst (bf16 slice) (+)= src (fp32 dense [pixels, C])
__global__ void __launch_bounds__(kTrThreads) add_f32_to_bf16_kernel(const float* src, __nv_bfloat16* dst, int64_t dst_pitch, int64_t pixels,
                                                                    int C, int accumulate) {
  const int64_t total = pixels * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t px = i / C;
    __nv_bfloat16* d = dst + px * dst_pitch + c;
    float v = src[i];
    if (accumulate) v += __bfloat162float(*d);
    *d = __float2bfloat16_rn(v);
  }
}

// ---------------------------------------------------------------------------------- stem wgrad
// dW3[co][r][s][c] = sum_pixels dY3[p][co] * x[n, c, 2ho + r - 1, 2wo + s - 1]   (3x3 stride-2 branch)
// dW1[co][c]       = sum_pixels dY1[p][co] * x[n, c, 2ho, 2wo]                    (1x1 stride-2 branch of a RepVGG stem)
// Persistent blocks walk 8x32 output tiles: the input patch (3 x 17 x 65 fp32) and the dY tile(s) are staged in
// shared memory, thread (tap group, co) accumulates its <= 7 taps over the 256 pixels in registers; one fp32
// atomic per (block, output) at the very end.
constexpr int kSwTH = 8, kSwTW = 32, kSwPH = 2 * kSwTH + 1, kSwPW = 2 * kSwTW + 1, kSwMaxTaps = 7;
constexpr int kSwPatchFloats = (3 * kSwPH * (kSwPW + 1) + 3) & ~3;      // keeps the dY tiles 16-byte aligned
__global__ void __launch_bounds__(kTrThreads) stem_wgrad_kernel(const void* x, int x_u8, float in_scale, View dy3, View dy1, int N, int H,
                                                               int W, int Cout, float* dw3, float* dw1) {
  extern __shared__ float sw_smem[];
  float* patch = sw_smem;                                               // [3][kSwPH][kSwPW + 1]
  __nv_bfloat16* g3 = reinterpret_cast<__nv_bfloat16*>(patch + kSwPatchFloats);   // [256][Cout]
  __nv_bfloat16* g1 = g3 + kSwTH * kSwTW * Cout;                        // [256][Cout] (only when dy1 is given)
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int tiles_w = (Wo + kSwTW - 1) / kSwTW, tiles_h = (Ho + kSwTH - 1) / kSwTH;
  const int64_t tiles = (int64_t)N * tiles_h * tiles_w;
  const int groups = blockDim.x / Cout;                                 // tap groups
  const int co = threadIdx.x % Cout, grp = threadIdx.x / Cout;
  const bool active = grp < groups;
  const bool has1 = dy1.p != nullptr;
  float acc[kSwMaxTaps], acc1 = 0.f;
  int off[kSwMaxTaps];                                                  // patch offset of my taps (-1 = none)
  int centre_i = -1, centre_off = 0;                                    // my centre tap (r = s = 1), if any: feeds dW1 as well
#pragma unroll
  for (int i = 0; i < kSwMaxTaps; ++i) {
    acc[i] = 0.f;
    const int k = grp + i * groups;                                     // k = (r*3 + s)*3 + c
    off[i] = -1;
    if (active && k < 27) {
      const int r = k / 9, sx = (k / 3) % 3, c = k % 3;
      off[i] = (c * kSwPH + r) * (kSwPW + 1) + sx;
      if (r == 1 && sx == 1) { centre_i = i; centre_off = off[i]; }
    }
  }
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int tw = (int)(t % tiles_w), th = (int)((t / tiles_w) % tiles_h), n = (int)(t / ((int64_t)tiles_w * tiles_h));
    const int ho0 = th * kSwTH, wo0 = tw * kSwTW;
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * kSwPH * kSwPW; i += blockDim.x) {
      const int pc = i % kSwPW, pr = (i / kSwPW) % kSwPH, c = i / (kSwPW * kSwPH);
      const int hi = 2 * ho0 - 1 + pr, wi = 2 * wo0 - 1 + pc;
      float v = 0.f;
      if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
        const int64_t idx = (((int64_t)n * 3 + c) * H + hi) * W + wi;
        v = x_u8 ? (float)reinterpret_cast<const uint8_t*>(x)[idx] * in_scale : reinterpret_cast<const float*>(x)[idx];
      }
      patch[(c * kSwPH + pr) * (kSwPW + 1) + pc] = v;
    }
    const int vec = Cout / 8;                                           // 16-byte chunks per pixel
    for (int i = threadIdx.x; i < kSwTH * kSwTW * vec; i += blockDim.x) {
      const int j = i % vec, px = i / vec;
      const int ho = ho0 + px / kSwTW, wo = wo0 + px % kSwTW;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (ho < Ho && wo < Wo) {
        const int64_t gp = ((int64_t)n * Ho + ho) * Wo + wo;
        a = *reinterpret_cast<const uint4*>(dy3.p + gp * dy3.pitch + j * 8);
        if (has1) b = *reinterpret_cast<const uint4*>(dy1.p + gp * dy1.pitch + j * 8);
      }
      *reinterpret_cast<uint4*>(g3 + (size_t)px * Cout + j * 8) = a;
      if (has1) *reinterpret_cast<uint4*>(g1 + (size_t)px * Cout + j * 8) = b;
    }
    __syncthreads();
    if (!active) continue;
    for (int py = 0; py < kSwTH; ++py) {
#pragma unroll 4
      for (int pxx = 0; pxx < kSwTW; ++pxx) {
        const int px = py * kSwTW + pxx;
        const float g = __bfloat162float(g3[(size_t)px * Cout + co]);
        const float* pp = patch + (2 * py) * (kSwPW + 1) + 2 * pxx;
#pragma unroll
        for (int i = 0; i < kSwMaxTaps; ++i)
          if (off[i] >= 0) acc[i] += g * pp[off[i]];
        if (has1 && centre_i >= 0) acc1 += __bfloat162float(g1[(size_t)px * Cout + co]) * pp[centre_off];
      }
    }
  }
  if (!active) return;
#pragma unroll
  for (int i = 0; i < kSwMaxTaps; ++i) {
    const int k = grp + i * groups;
    if (off[i] >= 0) atomicAdd(&dw3[co * 27 + k], acc[i]);
    if (has1 && i == centre_i) atomicAdd(&dw1[co * 3 + (k % 3)], acc1);
  }
}

// ---------------------------------------------------------------------------------- stem im2col (for the stem's weight gradient)
// patches[n, ho, wo, (r*3+s)*3 + c] = x[n, c, 2ho + r - 1, 2wo + s - 1] (zero outside the image), channels 27..31 zero, bf16.
// The stem's weight gradient is then an ordinary 1x1 wgrad GEMM over (patches, dY) on the tensor cores
// (K = all output pixels, M = Cout, N = 32), instead of 27 * Cout dot products of length N*Ho*Wo on CUDA cores.
__global__ void __launch_bounds__(256) stem_im2col_kernel(const void* x, int x_u8, float in_scale, int N, int H, int W, __nv_bfloat16* out,
                                                          __nv_bfloat16* out_lo) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t total = (int64_t)N * Ho * Wo;
  for (int64_t px = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; px < total; px += (int64_t)gridDim.x * blockDim.x) {
    const int wo = (int)(px % Wo), ho = (int)((px / Wo) % Ho), n = (int)(px / ((int64_t)Wo * Ho));
    float v[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = 2 * ho - 1 + r;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int sx = 0; sx < 3; ++sx) {
        const int wi = 2 * wo - 1 + sx;
        if (wi < 0 || wi >= W) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int64_t idx = (((int64_t)n * 3 + c) * H + hi) * W + wi;
          v[(r * 3 + sx) * 3 + c] = x_u8 ? (float)reinterpret_cast<const uint8_t*>(x)[idx] * in_scale : reinterpret_cast<const float*>(x)[idx];
        }
      }
    }
    __nv_bfloat16* o = out + px * 32;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float t[8] = {v[8 * j], v[8 * j + 1], v[8 * j + 2], v[8 * j + 3], v[8 * j + 4], v[8 * j + 5], v[8 * j + 6], v[8 * j + 7]};
      st8(o + 8 * j, t);
    }
    if (out_lo != nullptr) {      // residual plane: image = hi + lo to ~2^-17, so the gradient sees the fp32 image, not its bf16 rounding
      __nv_bfloat16* ol = out_lo + px * 32;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float t[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) t[k] = v[8 * j + k] - __bfloat162float(__float2bfloat16_rn(v[8 * j + k]));
        st8(ol + 8 * j, t);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- table-driven repack
// dst[d0][d1][d2][d3] (arbitrary strides) (+)= cast(src[d0][d1][d2][d3] (arbitrary, possibly negative strides)).
// One launch repacks every parameter of the network: fp32 master weights -> bf16 KRSC forward weights, rotated /
// transposed / parity-split dgrad weights, padded biases (per optimizer step), and -- in the other direction --
// fp32 KRSC weight gradients and float64 BatchNorm sums -> the flat fp32 gradient buffer in the reference's
// parameter layouts.
__global__ void __launch_bounds__(256) xform_kernel(const yv6_xform_seg* segs, const int32_t* chunk_seg, const int32_t* chunk_first,
                                                    int accumulate) {
  const int si = chunk_seg[blockIdx.x];
  const yv6_xform_seg sg = segs[si];
  const int64_t total = (int64_t)sg.n[0] * sg.n[1] * sg.n[2] * sg.n[3];
  const int64_t begin = (int64_t)(blockIdx.x - chunk_first[si]) * YV6_XFORM_CHUNK;
  const int64_t end = min(total, begin + YV6_XFORM_CHUNK);
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    int64_t r = i;
    const int d3 = (int)(r % sg.n[3]); r /= sg.n[3];
    const int d2 = (int)(r % sg.n[2]); r /= sg.n[2];
    const int d1 = (int)(r % sg.n[1]); r /= sg.n[1];
    const int d0 = (int)r;
    const int64_t so = (int64_t)d0 * sg.ss[0] + (int64_t)d1 * sg.ss[1] + (int64_t)d2 * sg.ss[2] + (int64_t)d3 * sg.ss[3];
    const int64_t dofs = (int64_t)d0 * sg.ds[0] + (int64_t)d1 * sg.ds[1] + (int64_t)d2 * sg.ds[2] + (int64_t)d3 * sg.ds[3];
    float v;
    if (sg.src_dtype == YV6_XF_F64) v = (float)reinterpret_cast<const double*>(sg.src)[so];
    else v = reinterpret_cast<const float*>(sg.src)[so];
    if (sg.dst_dtype == YV6_XF_BF16) {
      reinterpret_cast<__nv_bfloat16*>(sg.dst)[dofs] = __float2bfloat16_rn(v);
    } else {
      float* d = reinterpret_cast<float*>(sg.dst) + dofs;
      *d = accumulate ? (*d + v) : v;
    }
  }
}

// ---------------------------------------------------------------------------------- fused optimizer step
// torch.optim.SGD(momentum, nesterov=True) over the three parameter groups of build_optimizer (solver/build.py:10-33:
// BN weights / conv weights with weight decay / biases) and the ModelEMA update (utils/ema.py:28-37) in ONE pass over
// the flat fp32 parameter / gradient / momentum / EMA buffers.  Hyper-parameters come from device memory so that a
// captured CUDA graph follows the learning-rate schedule:
//   hyper = [lr_bnw, lr_w, lr_b, momentum, weight_decay (group w only), ema_decay, first_step, grad_scale]
__global__ void __launch_bounds__(256) sgd_ema_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ mom,
                                                      float* __restrict__ ema, const uint8_t* __restrict__ group, int64_t n4,
                                                      const float* __restrict__ hyper) {
  const float lr[3] = {__ldg(hyper), __ldg(hyper + 1), __ldg(hyper + 2)};
  const float mu = __ldg(hyper + 3), wd = __ldg(hyper + 4), d = __ldg(hyper + 5), gs = __ldg(hyper + 7);
  const bool first = __ldg(hyper + 6) != 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int gidx = group[i];                                          // one group id per 4 elements (segments are 16-byte aligned)
    float4 p = reinterpret_cast<float4*>(param)[i];
    if (gidx < 3) {
      const float4 g4 = reinterpret_cast<const float4*>(grad)[i];
      float4 b = first ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<float4*>(mom)[i];
      const float w = (gidx == 1) ? wd : 0.f, l = lr[gidx];
      float pe[4] = {p.x, p.y, p.z, p.w}, ge[4] = {g4.x, g4.y, g4.z, g4.w}, be[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float g = ge[j] * gs + w * pe[j];
        be[j] = first ? g : (mu * be[j] + g);
        g += mu * be[j];                                                // nesterov
        pe[j] -= l * g;
      }
      p = make_float4(pe[0], pe[1], pe[2], pe[3]);
      reinterpret_cast<float4*>(param)[i] = p;
      reinterpret_cast<float4*>(mom)[i] = make_float4(be[0], be[1], be[2], be[3]);
    }
    if (ema != nullptr && gidx < 4) {                                   // group 3 = float buffers (running statistics): EMA only
      float4 e = reinterpret_cast<float4*>(ema)[i];
      e.x = e.x * d + (1.f - d) * p.x; e.y = e.y * d + (1.f - d) * p.y;
      e.z = e.z * d + (1.f - d) * p.z; e.w = e.w * d + (1.f - d) * p.w;
      reinterpret_cast<float4*>(ema)[i] = e;
    }
  }
}

}  // namespace yv6

using namespace yv6;

static inline unsigned grid_for(int64_t total, int threads, int num_sms) {
  const int64_t want = (total + threads - 1) / threads;
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)num_sms * 16));
}

extern "C" int yv6_bn_stats(yv6_handle* h, const void* x, int64_t pixels, int32_t C, int64_t pitch, double* sum, double* sumsq,
                            void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && x && sum && sumsq, "bn_stats: null argument");
  YV6_REQUIRE(C % 8 == 0 && C <= 2048 && pitch % 8 == 0, "bn_stats: C=%d pitch=%lld", C, (long long)pitch);
  const int cgs = C / 8;
  int rows = std::max(1, kTrThreads / cgs);
  const int threads = cgs * rows;
  YV6_REQUIRE(threads <= 1024, "bn_stats: too many channels");
  cudaStream_t s = (cudaStream_t)stream;
  YV6_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * C, s));
  YV6_CHECK_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(double) * C, s));
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((pixels + rows - 1) / rows, (int64_t)h->num_sms * 8));
  bn_stats_kernel<<<grid, threads, sizeof(double) * 2 * C, s>>>(View{reinterpret_cast<const __nv_bfloat16*>(x), pitch}, pixels, C, sum, sumsq);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_bn_finalize(yv6_handle* h, const double* sum, const double* sumsq, double count, const float* gamma,
                               const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                               float* mean_out, float* invstd_out, float* scale, float* shift, int32_t C, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && sum && sumsq && gamma && beta && mean_out && invstd_out && scale && shift, "bn_finalize: null argument");
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sum, sumsq, count, gamma, beta, eps, momentum, running_mean,
                                                                      running_var, mean_out, invstd_out, scale, shift, C);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

static inline int chan_threads(int C) {
  const int cgs = C / 8;
  return cgs * std::max(1, kTrThreads / cgs);
}
static inline unsigned chan_grid(int64_t pixels, int C, int num_sms, int per_sm, int min_iters = 1) {
  // min_iters: pixels each thread should at least loop over (the reduction kernels pay per-block costs -- shared-memory
  // column sums, 2C..8C float64 atomics on the same addresses, the last-block pass -- that a small tensor cannot amortise
  // over hundreds of blocks)
  const int64_t rows = (int64_t)std::max(1, kTrThreads / (C / 8)) * min_iters;
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((pixels + rows - 1) / rows, (int64_t)num_sms * per_sm));
}
static int configure_train(yv6_handle* h) {
  if (h->configured & YV6_CFG_BN) return YV6_OK;
  YV6_CHECK_CUDA(cudaFuncSetAttribute(stem_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
  h->configured |= YV6_CFG_BN;
  return YV6_OK;
}

extern "C" int yv6_bn_stats_finalize(yv6_handle* h, const yv6_bn_stats_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->nb >= 1 && d->nb <= 3 && d->sums && d->counter, "bn_stats_finalize: bad descriptor");
  YV6_REQUIRE(d->C % 8 == 0 && d->C >= 8 && d->C <= 2048, "bn_stats_finalize: C=%d (multiple of 8, <= 2048)", d->C);
  StatsParams p;
  memset(&p, 0, sizeof(p));
  for (int b = 0; b < d->nb; ++b) {
    YV6_REQUIRE(d->x[b] && d->x_pitch[b] % 8 == 0, "bn_stats_finalize: branch %d input", b);
    YV6_REQUIRE(!d->stats[b] || (d->gamma[b] && d->beta[b]), "bn_stats_finalize: branch %d affine parameters", b);
    p.x[b] = View{reinterpret_cast<const __nv_bfloat16*>(d->x[b]), d->x_pitch[b]};
    p.gamma[b] = d->gamma[b]; p.beta[b] = d->beta[b]; p.rmean[b] = d->running_mean[b]; p.rvar[b] = d->running_var[b];
    p.stats[b] = d->stats[b];
  }
  p.nb = d->nb; p.C = d->C; p.pixels = d->pixels; p.sums = d->sums; p.counter = d->counter; p.eps = d->eps; p.momentum = d->momentum;
  cudaStream_t s = (cudaStream_t)stream;
  if (!d->zeroed) {
    YV6_CHECK_CUDA(cudaMemsetAsync(d->sums, 0, sizeof(double) * 2 * d->nb * d->C, s));
    YV6_CHECK_CUDA(cudaMemsetAsync(d->counter, 0, sizeof(unsigned int), s));
  }
  const int threads = chan_threads(d->C);
  const unsigned grid = chan_grid(d->pixels, d->C, h->num_sms, 4, 16);
  const size_t smem = sizeof(float) * (size_t)(threads / (d->C / 8)) * d->C;
  if (d->nb == 1) bn_stats_multi_kernel<1><<<grid, threads, smem, s>>>(p);
  else if (d->nb == 2) bn_stats_multi_kernel<2><<<grid, threads, smem, s>>>(p);
  else bn_stats_multi_kernel<3><<<grid, threads, smem, s>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_bn_apply_fwd(yv6_handle* h, const yv6_bn_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->nb >= 1 && d->nb <= 3 && d->y, "bn_apply_fwd: bad descriptor");
  YV6_REQUIRE(d->C % 8 == 0 && d->C >= 8 && d->C <= 2048, "bn_apply_fwd: C must be a multiple of 8, <= 2048");
  ApplyParams p;
  memset(&p, 0, sizeof(p));
  for (int b = 0; b < d->nb; ++b) {
    p.x[b] = View{reinterpret_cast<const __nv_bfloat16*>(d->x[b]), d->x_pitch[b]};
    p.scale[b] = d->scale[b];
    p.shift[b] = d->shift[b];
  }
  p.nb = d->nb; p.act = d->act; p.C = d->C; p.pixels = d->pixels;
  p.y = reinterpret_cast<__nv_bfloat16*>(d->y); p.y_pitch = d->y_pitch;
  p.res = View{reinterpret_cast<const __nv_bfloat16*>(d->res), d->res_pitch};
  p.alpha = d->res_alpha;
  p.alpha_dev = d->res_alpha_dev;
  const int threads = chan_threads(d->C);
  const unsigned grid = chan_grid(d->pixels, d->C, h->num_sms, 16, 2);
  cudaStream_t s = (cudaStream_t)stream;
  if (d->nb == 1) bn_apply_fwd_kernel<1><<<grid, threads, 0, s>>>(p);
  else if (d->nb == 2) bn_apply_fwd_kernel<2><<<grid, threads, 0, s>>>(p);
  else bn_apply_fwd_kernel<3><<<grid, threads, 0, s>>>(p);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_bn_bwd(yv6_handle* h, const yv6_bn_desc* d, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && d && d->nb >= 1 && d->nb <= 3 && d->dy && d->s1, "bn_bwd: bad descriptor");
  YV6_REQUIRE(d->C % 8 == 0 && d->C >= 8 && d->C <= 2048, "bn_bwd: C");
  BwdParams p;
  memset(&p, 0, sizeof(p));
  for (int b = 0; b < d->nb; ++b) {
    p.x[b] = View{reinterpret_cast<const __nv_bfloat16*>(d->x[b]), d->x_pitch[b]};
    p.mean[b] = d->mean[b]; p.invstd[b] = d->invstd[b]; p.scale[b] = d->scale[b]; p.shift[b] = d->shift[b];
    p.s2[b] = d->s2[b];
    p.dx[b] = reinterpret_cast<__nv_bfloat16*>(d->dx[b]); p.dx_pitch[b] = d->dx_pitch[b]; p.accumulate[b] = d->accumulate[b];
  }
  p.dy = View{reinterpret_cast<const __nv_bfloat16*>(d->dy), d->dy_pitch};
  p.res = View{reinterpret_cast<const __nv_bfloat16*>(d->res), d->res_pitch};
  p.alpha = d->res_alpha;
  p.alpha_dev = d->res_alpha_dev;
  p.dres = d->res ? reinterpret_cast<__nv_bfloat16*>(d->dres) : nullptr;
  p.dres_pitch = d->dres_pitch;
  p.dres_assign = d->dres_assign;
  p.dalpha = d->res ? d->dalpha : nullptr;
  YV6_REQUIRE(!d->res || (d->dres && d->dalpha), "bn_bwd: shortcut without dres / dalpha");
  p.nb = d->nb; p.act = d->act; p.C = d->C; p.pixels = d->pixels;
  p.s1 = d->s1;
  p.inv_count = 1.0 / (double)d->pixels;
  cudaStream_t s = (cudaStream_t)stream;
  // scratch of the two-pass scheme: caller-provided (training engine: one arena zeroed once per step) or the handle's
  if (d->work != nullptr) {
    YV6_REQUIRE(d->counter && d->coef, "bn_bwd: work without counter / coef");
    p.work = d->work; p.counter = d->counter; p.coef = d->coef;
  } else {
    char* base = reinterpret_cast<char*>(h->scratch);
    p.work = reinterpret_cast<double*>(base);
    p.coef = reinterpret_cast<float*>(base + sizeof(double) * 3 * 2048);
    p.counter = reinterpret_cast<unsigned int*>(base + sizeof(double) * 3 * 2048 + sizeof(float) * 6 * 2048);
  }
  if (d->work == nullptr || !d->zeroed) {
    YV6_CHECK_CUDA(cudaMemsetAsync(d->s1, 0, sizeof(double) * d->C, s));
    YV6_CHECK_CUDA(cudaMemsetAsync(p.work, 0, sizeof(double) * d->nb * d->C, s));
    YV6_CHECK_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(unsigned int), s));
    if (p.dalpha) YV6_CHECK_CUDA(cudaMemsetAsync(p.dalpha, 0, sizeof(double), s));
  }
  const int threads = chan_threads(d->C);
  const size_t smem = sizeof(float) * (size_t)(threads / (d->C / 8)) * d->C;
  const unsigned grid_r = chan_grid(d->pixels, d->C, h->num_sms, 4, 16), grid_a = chan_grid(d->pixels, d->C, h->num_sms, 16, 2);
  if (d->nb == 1) {
    bn_bwd_reduce_kernel<1><<<grid_r, threads, smem, s>>>(p);
    bn_bwd_apply_kernel<1><<<grid_a, threads, 0, s>>>(p);
  } else if (d->nb == 2) {
    bn_bwd_reduce_kernel<2><<<grid_r, threads, smem, s>>>(p);
    bn_bwd_apply_kernel<2><<<grid_a, threads, 0, s>>>(p);
  } else {
    bn_bwd_reduce_kernel<3><<<grid_r, threads, smem, s>>>(p);
    bn_bwd_apply_kernel<3><<<grid_a, threads, 0, s>>>(p);
  }
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_head_grad_prep(yv6_handle* h, const float* grad, const float* scores_or_null, int32_t B, int32_t A, int32_t ch,
                                  int32_t level_off, int32_t level_hw, int32_t ch_pad, void* out_bf16, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && grad && out_bf16 && ch_pad >= ch, "head_grad_prep: bad argument");
  const int64_t total = (int64_t)B * level_hw * ch_pad;
  head_grad_prep_kernel<<<grid_for(total, kTrThreads, h->num_sms), kTrThreads, 0, (cudaStream_t)stream>>>(
      grad, scores_or_null, B, A, ch, level_off, level_hw, ch_pad, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_maxpool5_bwd(yv6_handle* h, const void* x, int64_t x_pitch, const void* dy, int64_t dy_pitch, int32_t N,
                                int32_t H, int32_t W, int32_t C, float* dx_scratch, void* dx, int64_t dx_pitch, int32_t accumulate,
                                void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && x && dy && dx_scratch && dx, "maxpool5_bwd: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t total = (int64_t)N * H * W * C;
  YV6_CHECK_CUDA(cudaMemsetAsync(dx_scratch, 0, sizeof(float) * total, s));
  maxpool5_bwd_kernel<<<grid_for(total, kTrThreads, h->num_sms), kTrThreads, 0, s>>>(
      View{reinterpret_cast<const __nv_bfloat16*>(x), x_pitch}, View{reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch}, N, H, W, C,
      dx_scratch);
  add_f32_to_bf16_kernel<<<grid_for(total, kTrThreads, h->num_sms), kTrThreads, 0, s>>>(
      dx_scratch, reinterpret_cast<__nv_bfloat16*>(dx), dx_pitch, (int64_t)N * H * W, C, accumulate);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_stem_wgrad2(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, const void* dy3, int64_t dy3_pitch,
                               const void* dy1, int64_t dy1_pitch, int32_t N, int32_t H, int32_t W, int32_t Cout, float* dw3, float* dw1,
                               int32_t zeroed, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && x && dy3 && dw3 && Cout >= 8 && Cout <= 64 && Cout % 8 == 0, "stem_wgrad: bad argument");
  YV6_REQUIRE(dy3_pitch % 8 == 0 && (!dy1 || (dw1 && dy1_pitch % 8 == 0)), "stem_wgrad: dY pitch / dW1");
  if (int rc = configure_train(h)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (!zeroed) {
    YV6_CHECK_CUDA(cudaMemsetAsync(dw3, 0, sizeof(float) * 27 * Cout, s));
    if (dy1) YV6_CHECK_CUDA(cudaMemsetAsync(dw1, 0, sizeof(float) * 3 * Cout, s));
  }
  const int threads = (kTrThreads / Cout) * Cout;
  const size_t smem = sizeof(float) * kSwPatchFloats + (size_t)(dy1 ? 2 : 1) * kSwTH * kSwTW * Cout * sizeof(__nv_bfloat16);
  stem_wgrad_kernel<<<h->num_sms * 2, threads, smem, s>>>(x, x_dtype == YV6_DT_U8, in_scale,
                                                          View{reinterpret_cast<const __nv_bfloat16*>(dy3), dy3_pitch},
                                                          View{reinterpret_cast<const __nv_bfloat16*>(dy1), dy1_pitch}, N, H, W, Cout, dw3, dw1);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_stem_wgrad(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, const void* dy, int64_t dy_pitch,
                              int32_t N, int32_t H, int32_t W, int32_t Cout, float* dw, void* stream) {
  return yv6_stem_wgrad2(h, x, x_dtype, in_scale, dy, dy_pitch, nullptr, 0, N, H, W, Cout, dw, nullptr, 0, stream);
}

extern "C" int yv6_stem_im2col(yv6_handle* h, const void* x, int32_t x_dtype, float in_scale, int32_t N, int32_t H, int32_t W,
                               void* patches_bf16, void* patches_lo_bf16, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && x && patches_bf16 && N > 0 && H > 0 && W > 0, "stem_im2col: bad argument");
  const int64_t total = (int64_t)N * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1);
  stem_im2col_kernel<<<grid_for(total, 256, h->num_sms), 256, 0, (cudaStream_t)stream>>>(x, x_dtype == YV6_DT_U8, in_scale, N, H, W,
                                                                                         reinterpret_cast<__nv_bfloat16*>(patches_bf16),
                                                                                         reinterpret_cast<__nv_bfloat16*>(patches_lo_bf16));
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_xform(yv6_handle* h, const yv6_xform_seg* segs_dev, const int32_t* chunk_seg_dev, const int32_t* chunk_first_dev,
                         int32_t n_chunks, int32_t accumulate, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && segs_dev && chunk_seg_dev && chunk_first_dev && n_chunks >= 0, "xform: bad argument");
  if (n_chunks == 0) return YV6_OK;
  xform_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>(segs_dev, chunk_seg_dev, chunk_first_dev, accumulate);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_sgd_ema_step(yv6_handle* h, float* param, const float* grad, float* momentum_buf, float* ema_or_null,
                                const uint8_t* group_per4, int64_t n, const float* hyper_dev, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && param && grad && momentum_buf && group_per4 && hyper_dev && n >= 0 && n % 4 == 0, "sgd_ema_step: bad argument");
  if (n == 0) return YV6_OK;
  const int64_t n4 = n / 4;
  const unsigned grid = (unsigned)std::min<int64_t>((n4 + 255) / 256, (int64_t)h->num_sms * 16);
  sgd_ema_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(param, grad, momentum_buf, ema_or_null, group_per4, n4, hyper_dev);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
