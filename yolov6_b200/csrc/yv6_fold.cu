// yv6_fold.cu -- the inference weight fold on the device (include/yv6.h, "Inference weight fold"): fold.py's BatchNorm folding
// and RepVGG / QARepVGG re-parameterisation, and the engine's operand casts, from the train-form state in a flat fp32 buffer
// straight into the weight tensors of a built InferEngine.
//
//   fold_chan_kernel : one CTA per op, one thread per output channel: the float64 BatchNorm affine of each branch
//                      (scale = gamma / sqrt(var + 1e-3), shift = beta - mean * scale) and the folded bias.
//   fold_elem_kernel : YV6_FOLD_CHUNK elements of one record per CTA: the float64 weight of domain point (o, r, s, c), then the
//                      record's cast (fp32, bf16, fp16 or three bf16 planes), or in check mode the fp16 range check.
//
// Every float64 operation is an explicit round-to-nearest intrinsic in fold.py's operation order, so nothing is contracted into
// an FMA and every add fold.py performs happens here too -- including `k3 + pad(k1)` at the off-centre taps, where
// -0.0 + 0.0 = +0.0 changes the stored bits.  Casts follow torch's CPU path: float64 -> fp32 (round to nearest) first, then
// bf16 / fp16 round to nearest even (torch converts float64 to fp16 through fp32).  The split3 residuals are fp32 subtractions,
// as in ops.split3.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace {

constexpr double BN_EPS = 1e-3;     // fold.BN_EPS (torch_utils.py:41-43)

__device__ __forceinline__ void bn_affine(const float* flat, const int64_t* bn, int o, double& scale, double& shift) {
  const double g = (double)flat[bn[0] + o], b = (double)flat[bn[1] + o];
  const double m = (double)flat[bn[2] + o], v = (double)flat[bn[3] + o];
  scale = __ddiv_rn(g, __dsqrt_rn(__dadd_rn(v, BN_EPS)));
  shift = __dsub_rn(b, __dmul_rn(m, scale));
}

__global__ void __launch_bounds__(256) fold_chan_kernel(const float* __restrict__ flat, const yv6_fold_chan* __restrict__ chans,
                                                        double* __restrict__ coef) {
  const yv6_fold_chan ch = chans[blockIdx.x];
  for (int o = threadIdx.x; o < ch.n; o += blockDim.x) {
    double A = 1.0, B = 1.0, D = 0.0, P = 1.0, bias = 0.0, s0, t0, s1, t1;
    switch (ch.layout) {
      case YV6_FOLD_C_DP:        // scale * (conv + b) + shift
        bn_affine(flat, ch.bn[0], o, s0, t0);
        A = s0;
        bias = __dadd_rn(__dmul_rn((double)flat[ch.b + o], s0), t0);
        break;
      case YV6_FOLD_C_REP:       // b3 + b1 (+ shift of the identity BatchNorm)
        bn_affine(flat, ch.bn[0], o, s0, t0);
        bn_affine(flat, ch.bn[1], o, s1, t1);
        A = s0, B = s1;
        bias = __dadd_rn(t0, t1);
        if (ch.bn[2][0] >= 0) {
          double s2, t2;
          bn_affine(flat, ch.bn[2], o, s2, t2);
          D = s2;
          bias = __dadd_rn(bias, t2);
        }
        break;
      case YV6_FOLD_C_QA:        // b_dense * scale_post + shift_post
        bn_affine(flat, ch.bn[0], o, s0, t0);
        bn_affine(flat, ch.bn[1], o, s1, t1);
        A = s0, P = s1;
        bias = __dadd_rn(__dmul_rn(t0, s1), t1);
        break;
      case YV6_FOLD_C_BN:
        bn_affine(flat, ch.bn[0], o, s0, t0);
        A = s0, bias = t0;
        break;
      default:                   // C_BIAS
        bias = (double)flat[ch.b + o];
        break;
    }
    double* c = coef + ch.coef + 5 * (int64_t)o;
    c[0] = A, c[1] = B, c[2] = D, c[3] = P, c[4] = bias;
  }
}

__device__ __forceinline__ double fold_value(const yv6_fold_rec& R, const float* __restrict__ flat, const double* __restrict__ coef,
                                             int o, int r, int s, int c) {
  const int rs = r + R.r0, ss = s + R.s0;
  const double* cf = coef + R.coef + 5 * (int64_t)o;
  switch (R.layout) {
    case YV6_FOLD_BIAS: return cf[4];
    case YV6_FOLD_COPY: return (double)flat[R.w + o];
    case YV6_FOLD_W_CONVT: return (double)flat[R.w + (((int64_t)c * R.cout + o) * 2 + rs) * 2 + ss];
    default: break;
  }
  const double w = (double)flat[R.w + (((int64_t)o * R.cin + c) * R.k + rs) * R.k + ss];
  const bool center = rs == 1 && ss == 1, diag = (R.flags & YV6_FOLD_IDENTITY) && o == c;
  switch (R.layout) {
    case YV6_FOLD_W_COPY: return w;
    case YV6_FOLD_W_REP: {
      double t = __dadd_rn(__dmul_rn(w, cf[0]), center ? __dmul_rn((double)flat[R.w1 + (int64_t)o * R.cin + c], cf[1]) : 0.0);
      if (diag && center) t = __dadd_rn(t, cf[2]);
      return t;
    }
    case YV6_FOLD_W_QA: {
      double t = __dadd_rn(__dmul_rn(w, cf[0]), center ? (double)flat[R.w1 + (int64_t)o * R.cin + c] : 0.0);
      if (diag) {
        if (center) t = __dadd_rn(t, 1.0);
        if (R.flags & YV6_FOLD_AVG) t = __dadd_rn(t, 1.0 / 9.0);
      }
      return __dmul_rn(t, cf[3]);
    }
    default: return __dmul_rn(w, cf[0]);      // W
  }
}

__global__ void __launch_bounds__(256) fold_elem_kernel(const float* __restrict__ flat, const yv6_fold_rec* __restrict__ recs, int n_recs,
                                                        const double* __restrict__ coef, unsigned long long* __restrict__ checks,
                                                        int check_only) {
  int lo = 0, hi = n_recs - 1;              // the last record with blk0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (recs[mid].blk0 <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const yv6_fold_rec R = recs[lo];
  if (check_only && R.check < 0) return;
  const int64_t total = (int64_t)R.n[0] * R.n[1] * R.n[2] * R.n[3];
  const int64_t begin = ((int64_t)blockIdx.x - R.blk0) * YV6_FOLD_CHUNK;
  const int64_t end = min(total, begin + YV6_FOLD_CHUNK);
  bool bad = false;
  unsigned long long vmax = 0;
  for (int64_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
    int64_t q = i;
    const int c = (int)(q % R.n[3]); q /= R.n[3];
    const int s = (int)(q % R.n[2]); q /= R.n[2];
    const int r = (int)(q % R.n[1]); q /= R.n[1];
    const int o = (int)q;
    const double v = fold_value(R, flat, coef, o, r, s, c);
    const float f = __double2float_rn(v);
    if (check_only) {
      bad |= !isfinite(__half2float(__float2half_rn(f)));
      vmax = max(vmax, (unsigned long long)__double_as_longlong(fabs(v)));
      continue;
    }
    const int64_t d = (int64_t)o * R.ds[0] + (int64_t)r * R.ds[1] + (int64_t)s * R.ds[2] + (int64_t)c * R.ds[3];
    switch (R.fmt) {
      case YV6_FOLD_F32: reinterpret_cast<float*>(R.dst)[d] = f; break;
      case YV6_FOLD_BF16: reinterpret_cast<__nv_bfloat16*>(R.dst)[d] = __float2bfloat16_rn(f); break;
      case YV6_FOLD_F16: reinterpret_cast<__half*>(R.dst)[d] = __float2half_rn(f); break;
      default: {                            // SPLIT3
        __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(R.dst) + d;
        const __nv_bfloat16 p0 = __float2bfloat16_rn(f);
        const float r1 = __fsub_rn(f, __bfloat162float(p0));
        const __nv_bfloat16 p1 = __float2bfloat16_rn(r1);
        const float r2 = __fsub_rn(r1, __bfloat162float(p1));
        p[0] = p0, p[R.plane_stride] = p1, p[2 * R.plane_stride] = __float2bfloat16_rn(r2);
      }
    }
  }
  if (check_only) {
    if (bad) atomicOr(checks + 2 * R.check, 1ull);
    atomicMax(checks + 2 * R.check + 1, vmax);
  }
}

}  // namespace

extern "C" int yv6_fold(yv6_handle* h, const float* flat, const yv6_fold_chan* chans_dev, int32_t n_chans, const yv6_fold_rec* recs_dev,
                        int32_t n_recs, int64_t n_blocks, double* coef, unsigned long long* checks, int32_t check_only, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && flat && (n_chans == 0 || (chans_dev && coef)) && (n_recs == 0 || recs_dev) && n_chans >= 0 && n_recs >= 0 &&
              n_blocks >= 0 && n_blocks < (1ll << 31), "fold: bad argument");
  YV6_REQUIRE(!check_only || checks, "fold: check_only needs the checks buffer");
  if (n_chans > 0) {
    fold_chan_kernel<<<n_chans, 256, 0, (cudaStream_t)stream>>>(flat, chans_dev, coef);
    YV6_CHECK_CUDA(cudaGetLastError());
  }
  if (n_recs > 0 && n_blocks > 0) {
    fold_elem_kernel<<<(unsigned)n_blocks, 256, 0, (cudaStream_t)stream>>>(flat, recs_dev, n_recs, coef, checks, check_only);
    YV6_CHECK_CUDA(cudaGetLastError());
  }
  return YV6_OK;
}
