// yv6_metrics.cu -- the Evaler's precision / recall metric (do_pr_metric, yolov6/core/evaler.py:109-226) on the device.
//
//   yv6_pr_match  : one CTA per image of a batch.  Evaler.scale_coords of the NMS rows and of the labels (xywh2xyxy, times
//                   the letterboxed W / H), general.box_iou, the correct flags of metrics.process_batch at the ten IoU
//                   thresholds and ConfusionMatrix.process_batch; (conf, cls, correct bits) land in a fixed slot per image
//                   of the dataset, label / prediction counts and the matrix are integer atomics.
//   yv6_pr_metric : ap_per_class / compute_ap (metrics.py:13-102) and the Evaler's summary over every accumulated row:
//                   stable LSD radix sort of (class, descending conf) keys, one CTA per (class, threshold) for the running
//                   TP / FP counts, the precision envelope and the 101-point interpolated AP, one CTA per class for the
//                   1000-point P / R / F1 curves, one CTA for F1's mean, its arg-max and the means.
//
// process_batch's argsort / unique / unique (metrics.py:154-166) reduces to a rule: L(d) is the same-class label with the
// highest IoU (ties: lowest label index); d is correct at threshold t iff IoU(L(d), d) >= iouv[t] and no detection with a
// lower row index has the same L at t.  The second np.unique keeps the lowest detection index, not the highest IoU.
//
// All fp32 arithmetic that feeds a comparison and all fp64 arithmetic of the metric uses explicit round-to-nearest
// intrinsics in the reference's operation order, so flags, counts, curves and the arg-max are bit-exact; np.interp is
// restated exactly (a query on repeated sample points takes the last of them).
#include <algorithm>

#include "yv6_common.cuh"
#include "yv6_handle.h"
#include "yv6_scale_coords.cuh"
#include "yv6_sort.cuh"

namespace yv6 {

constexpr int kPrNiou = 10;
constexpr int kPrCurve = 1000;       // np.linspace(0, 1, 1000) of ap_per_class
constexpr int kPrAp = 101;           // np.linspace(0, 1, 101) of compute_ap
constexpr int kMatchThreads = 256;
constexpr int kApThreads = 256, kApItems = 8, kApChunk = kApThreads * kApItems;
enum { kPrErrLabelCls = 1, kPrErrDetCls = 2, kPrErrLabels = 4 };

__device__ __forceinline__ bool valid_cls(float c, int nc) { return c >= 0.f && c < (float)nc && c == floorf(c); }

// general.box_iou (general.py:64-86): inter / ((area_l + area_d) - inter)
__device__ __forceinline__ float box_iou_rn(float4 a, float4 b) {
  const float area1 = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float area2 = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  const float iw = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
}

// ------------------------------------------------------------------------------------------------
// per-image matching
// ------------------------------------------------------------------------------------------------
struct PrMatchArgs {
  yv6_pr_state st;
  const float* det;        // [B][D][6]
  const int32_t* count;    // [B]
  const float* targets;    // [n][6] (image, cls, x, y, w, h), normalised
  const float* meta;       // [B][6]
  const float* iouv;       // [10]
  int32_t D, n, H, W, first, lcap;
};

__global__ void __launch_bounds__(kMatchThreads) pr_match_kernel(PrMatchArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int D = a.D, nc = a.st.nc;
  float4* dbox = reinterpret_cast<float4*>(smem);
  float4* lbox = dbox + D;
  float* dconf = reinterpret_cast<float*>(lbox + a.lcap);
  float* dcls = dconf + D;
  float* cm = dcls + D;                                     // IoU of the confusion match
  int* dl = reinterpret_cast<int*>(cm + D);                 // L(d), -1 = none
  int* dmask = dl + D;                                      // thresholds at which L(d) is a candidate
  int* cl = dmask + D;                                      // confusion match label, -1 = none
  float* lcls = reinterpret_cast<float*>(cl + D);
  int* lwin = reinterpret_cast<int*>(lcls + a.lcap);
  __shared__ int s_wcnt[kMatchThreads / 32];
  __shared__ float s_iouv[kPrNiou];

  const int nd = min(max(a.count[b], 0), D);
  const int img = a.first + b;
  const float* m = a.meta + b * 6;
  if (tid < kPrNiou) s_iouv[tid] = a.iouv[tid];
  // labels of image b in their original order: targets[targets[:, 0] == b] (evaler.py:157)
  int nl = 0;
  for (int base = 0; base < a.n; base += kMatchThreads) {
    const int r = base + tid;
    const bool mine = r < a.n && a.targets[(int64_t)r * 6] == (float)b;
    const unsigned bal = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int w = 0; w < kMatchThreads / 32; ++w) {
      off += w < warp ? s_wcnt[w] : 0;
      tot += s_wcnt[w];
    }
    const int pos = nl + off + __popc(bal & ((1u << lane) - 1u));
    if (mine) {
      const float* t = a.targets + (int64_t)r * 6;
      const float c = t[1];
      if (!valid_cls(c, nc)) atomicOr(a.st.flags, kPrErrLabelCls);
      else atomicAdd(a.st.nt + (int)c, 1);
      if (pos < a.lcap) {
        // yolov6/utils/nms.py:21-28 xywh2xyxy, then x * W, y * H (evaler.py:178-180), then scale_coords
        const float x = t[2], y = t[3], hw = __fdiv_rn(t[4], 2.f), hh = __fdiv_rn(t[5], 2.f);
        const float fw = (float)a.W, fh = (float)a.H;
        lbox[pos] = scale_coords_rn(__fmul_rn(__fsub_rn(x, hw), fw), __fmul_rn(__fsub_rn(y, hh), fh), __fmul_rn(__fadd_rn(x, hw), fw),
                                    __fmul_rn(__fadd_rn(y, hh), fh), m);
        lcls[pos] = c;
        lwin[pos] = -1;
      } else {
        atomicOr(a.st.flags, kPrErrLabels);
      }
    }
    nl += tot;
    __syncthreads();
  }
  nl = min(nl, a.lcap);
  for (int j = tid; j < nd; j += kMatchThreads) {
    const float* r = a.det + ((int64_t)b * D + j) * 6;
    dbox[j] = scale_coords_rn(r[0], r[1], r[2], r[3], m);
    dconf[j] = r[4];
    dcls[j] = r[5];
    const int64_t slot = (int64_t)img * a.st.max_det + j;
    a.st.conf[slot] = r[4];
    a.st.cls[slot] = r[5];
    if (!valid_cls(r[5], nc)) atomicOr(a.st.flags, kPrErrDetCls);
    else atomicAdd(a.st.npred + (int)r[5], 1);
  }
  if (tid == 0) a.st.ndet[img] = nd;
  __syncthreads();
  const bool conf_on = a.st.confusion != 0 && nl > 0 && nd > 0;
  for (int j = tid; j < nd; j += kMatchThreads) {
    const float4 bx = dbox[j];
    const float c = dcls[j];
    const bool kept = conf_on && dconf[j] > 0.25f;            // ConfusionMatrix(conf=0.25) (metrics.py:171,187)
    int best = -1, cbest = -1;
    float biou = 0.f, ciou = 0.f;
    for (int l = 0; l < nl; ++l) {
      const float iou = box_iou_rn(lbox[l], bx);
      if (lcls[l] == c && iou >= s_iouv[0] && (best < 0 || iou > biou)) best = l, biou = iou;
      if (kept && iou > 0.45f && (cbest < 0 || iou > ciou)) cbest = l, ciou = iou;   // iou_thres=0.45, class-agnostic
    }
    int mask = 0;
    if (best >= 0)
      for (int t = 0; t < kPrNiou; ++t) mask |= (biou >= s_iouv[t]) << t;
    dl[j] = best;
    dmask[j] = mask;
    cl[j] = cbest;
    cm[j] = ciou;
  }
  __syncthreads();
  int any = 0;
  for (int j = tid; j < nd; j += kMatchThreads) {
    int bits = 0;
    const int L = dl[j];
    if (L >= 0) {
      int blocked = 0;
      for (int k = 0; k < j; ++k) blocked |= dl[k] == L ? dmask[k] : 0;
      bits = dmask[j] & ~blocked;
    }
    a.st.correct[(int64_t)img * a.st.max_det + j] = (uint16_t)bits;
    any |= bits;
  }
  if (any) atomicOr(a.st.flags + 1, 1);
  if (!conf_on) return;
  // ConfusionMatrix.process_batch (metrics.py:177-215): each kept detection keeps its best label, each label keeps the
  // detection with the highest IoU among those (ties: lowest index)
  bool matched = false;
  for (int j = tid; j < nd; j += kMatchThreads) {
    const int L = cl[j];
    if (L < 0) continue;
    matched = true;
    bool win = true;
    for (int k = 0; k < nd && win; ++k)
      if (k != j && cl[k] == L && (cm[k] > cm[j] || (cm[k] == cm[j] && k < j))) win = false;
    if (win) lwin[L] = j;
  }
  const bool any_match = __syncthreads_or(matched);
  const int ld = nc + 1;
  for (int l = tid; l < nl; l += kMatchThreads) {
    if (!valid_cls(lcls[l], nc)) continue;
    const int gc = (int)lcls[l], w = lwin[l];
    const int row = (any_match && w >= 0) ? (valid_cls(dcls[w], nc) ? (int)dcls[w] : -1) : nc;
    if (row >= 0) atomicAdd(a.st.matrix + row * ld + gc, 1);
  }
  if (!any_match) return;
  for (int j = tid; j < nd; j += kMatchThreads)
    if (dconf[j] > 0.25f && !(cl[j] >= 0 && lwin[cl[j]] == j) && valid_cls(dcls[j], nc)) atomicAdd(a.st.matrix + (int)dcls[j] * ld + nc, 1);
}

// ------------------------------------------------------------------------------------------------
// keys of the stable LSD radix sort (yv6_sort.cuh): (class << 32 | ~ordered(conf)) keys, 8-bit digits
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t conf_desc_bits(float f) {
  const uint32_t u = __float_as_uint(f);
  return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}
__device__ __forceinline__ float conf_of_key(uint64_t k) {
  const uint32_t o = ~(uint32_t)k;
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

__global__ void pr_keys_kernel(yv6_pr_state st, int64_t N, uint64_t* keys, uint32_t* vals) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  const int img = (int)(s / st.max_det), j = (int)(s - (int64_t)img * st.max_det);
  uint64_t k = ((uint64_t)st.nc << 32) | 0xffffffffull;        // empty slot: after every class
  if (j < st.ndet[img]) {
    const float c = st.cls[s];
    if (valid_cls(c, st.nc)) k = ((uint64_t)(uint32_t)c << 32) | conf_desc_bits(st.conf[s]);
  }
  keys[s] = k;
  vals[s] = (uint32_t)s;
}

// ------------------------------------------------------------------------------------------------
// per (class, threshold): running TP counts, precision envelope, 101-point interpolated AP (compute_ap)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int seg_start(const int32_t* npred, int c) {
  int s = 0;
  for (int k = 0; k < c; ++k) s += npred[k];
  return s;
}

struct PrMetricArgs {
  yv6_pr_state st;
  const uint64_t* keys;    // sorted
  const uint32_t* vals;    // sorted slots
  int32_t* tpc0;           // [N] running TP count at iouv[0], in sorted order
  const double* px;        // [1000]
  const double* x101;      // [101]
  double* out;
};

__device__ __forceinline__ double recall_of(int tpc, int nl) { return __ddiv_rn((double)tpc, __dadd_rn((double)nl, 1e-16)); }

__global__ void __launch_bounds__(kApThreads) pr_ap_kernel(PrMetricArgs a) {
  const int c = blockIdx.x, t = blockIdx.y, tid = threadIdx.x;
  const int nl = a.st.nt[c];
  if (nl == 0) return;
  const int n = a.st.npred[c], start = seg_start(a.st.npred, c);
  double* ap = a.out + (int64_t)a.st.nc * 3 * kPrCurve;
  if (n == 0) {
    if (tid == 0) ap[c * kPrNiou + t] = 0.0;
    return;
  }
  __shared__ int s_K[kPrAp], s_P[kPrAp], s_wi[32];
  __shared__ double s_x[kPrAp], s_Sa[kPrAp], s_Sb[kPrAp], s_y[kPrAp], s_wd[32];
  __shared__ double s_chunk[kApChunk];
  if (tid < kPrAp) {
    // K = the largest label count k whose recall k / (n_l + 1e-16) is <= x: the recall points at or below x are the rows
    // before the (K + 1)-th true positive
    const double x = a.x101[tid];
    int k = min(max((int)(x * nl), 0), nl);
    while (k < nl && recall_of(k + 1, nl) <= x) ++k;
    while (k > 0 && recall_of(k, nl) > x) --k;
    s_K[tid] = k;
    s_P[tid] = n;
    s_x[tid] = x;
  }
  __syncthreads();
  const uint16_t* corr = a.st.correct;
  int carry = 0;
  for (int cb = 0; cb < n; cb += kApChunk) {
    const int i0 = cb + tid * kApItems;
    int bits = 0, cnt = 0;
#pragma unroll
    for (int k = 0; k < kApItems; ++k) {
      const int i = i0 + k;
      const int tp = i < n ? (corr[a.vals[start + i]] >> t) & 1 : 0;
      bits |= tp << k;
      cnt += tp;
    }
    int tot;
    int tpc = carry + block_excl_sum(cnt, s_wi, &tot);
#pragma unroll
    for (int k = 0; k < kApItems; ++k) {
      const int i = i0 + k;
      if (i >= n) break;
      if ((bits >> k) & 1) {
        ++tpc;
        int lo = 0, hi = kPrAp;                               // first query with K + 1 >= tpc
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (s_K[mid] + 1 < tpc) lo = mid + 1;
          else hi = mid;
        }
        for (int q = lo; q < kPrAp && s_K[q] + 1 == tpc; ++q) s_P[q] = i;
      }
      if (t == 0) a.tpc0[start + i] = tpc;
    }
    carry += tot;
  }
  const int T = carry;
  __syncthreads();
  // reverse pass: suffix maximum of precision (the envelope) at the rows the queries need
  int after = 0;
  double cmax = 0.0;
  const int nchunks = (n + kApChunk - 1) / kApChunk;
  for (int ci = nchunks - 1; ci >= 0; --ci) {
    const int cb = ci * kApChunk, i0 = cb + tid * kApItems;
    int bits = 0, cnt = 0;
#pragma unroll
    for (int k = 0; k < kApItems; ++k) {
      const int i = i0 + k;
      const int tp = i < n ? (corr[a.vals[start + i]] >> t) & 1 : 0;
      bits |= tp << k;
      cnt += tp;
    }
    int tot;
    const int excl = block_excl_sum(cnt, s_wi, &tot);
    const int before = T - after - tot;
    double prec[kApItems];
    int tpc = before + excl;
    double tmax = 0.0;
#pragma unroll
    for (int k = 0; k < kApItems; ++k) {
      const int i = i0 + k;
      tpc += (bits >> k) & 1;
      prec[k] = i < n ? __ddiv_rn((double)tpc, (double)(i + 1)) : 0.0;   // tpc / (tpc + fpc)
      tmax = fmax(tmax, prec[k]);
    }
    double ctot;
    double run = fmax(block_excl_sufmax(tmax, s_wd, &ctot), cmax);
#pragma unroll
    for (int k = kApItems - 1; k >= 0; --k) {
      run = fmax(run, prec[k]);
      if (i0 + k < n) s_chunk[tid * kApItems + k] = run;
    }
    __syncthreads();
    if (tid < kPrAp) {
      const int P = s_P[tid];
      if (P - 1 >= cb && P - 1 < cb + kApChunk) s_Sa[tid] = s_chunk[P - 1 - cb];
      if (P < n && P >= cb && P < cb + kApChunk) s_Sb[tid] = s_chunk[P - cb];
    }
    after += tot;
    cmax = fmax(cmax, ctot);
    __syncthreads();
  }
  if (tid < kPrAp) {
    // np.interp(x, mrec, mpre): j = last index with mrec[j] <= x; mrec = [0, recall, recall[-1] + 0.01], mpre = envelope
    const double x = s_x[tid];
    const int P = s_P[tid], K = s_K[tid];
    double y;
    if (P == n) {
      const double rt = recall_of(T, nl), last = __dadd_rn(rt, 0.01), e = s_Sa[tid];
      if (last <= x) y = 0.0;
      else if (rt == x) y = e;
      else y = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(0.0, e), __dsub_rn(last, rt)), __dsub_rn(x, rt)), e);
    } else {
      const double mj = recall_of(K, nl), mj1 = recall_of(K + 1, nl);
      const double ej = P == 0 ? 1.0 : s_Sa[tid], ej1 = s_Sb[tid];
      if (mj == x) y = ej;
      else y = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(ej1, ej), __dsub_rn(mj1, mj)), __dsub_rn(x, mj)), ej);
    }
    s_y[tid] = y;
  }
  __syncthreads();
  if (tid == 0) {
    // np.trapz(y, x) = add.reduce(diff(x) * (y[1:] + y[:-1]) / 2.0), numpy's pairwise order for 100 terms
    double r[8];
    auto term = [&](int k) {
      return __ddiv_rn(__dmul_rn(__dsub_rn(s_x[k + 1], s_x[k]), __dadd_rn(s_y[k + 1], s_y[k])), 2.0);
    };
    for (int k = 0; k < 8; ++k) r[k] = term(k);
    int i = 8;
    for (; i < (kPrAp - 1) - (kPrAp - 1) % 8; i += 8)
      for (int k = 0; k < 8; ++k) r[k] = __dadd_rn(r[k], term(i + k));
    double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < kPrAp - 1; ++i) s = __dadd_rn(s, term(i));
    ap[c * kPrNiou + t] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// per class: P / R curves at iouv[0] on px = linspace(0, 1, 1000) and F1
//   r = interp(-px, -conf, recall, left=0), p = interp(-px, -conf, precision, left=1), f1 = 2 p r / (p + r + 1e-16)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pr_curve_kernel(PrMetricArgs a) {
  const int c = blockIdx.x, nl = a.st.nt[c];
  if (nl == 0) return;
  const int n = a.st.npred[c], start = seg_start(a.st.npred, c);
  if (n == 0) return;                                       // rows stay 0 (np.zeros)
  const int nc = a.st.nc;
  double* P = a.out + (int64_t)c * kPrCurve;
  double* R = P + (int64_t)nc * kPrCurve;
  double* F = R + (int64_t)nc * kPrCurve;
  const uint64_t* keys = a.keys + start;
  const int32_t* tpc = a.tpc0 + start;
  for (int m = threadIdx.x; m < kPrCurve; m += blockDim.x) {
    const double px = a.px[m], x = -px;
    int lo = 0, hi = n;                                     // rows with -conf <= -px
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (-(double)conf_of_key(keys[mid]) <= x) lo = mid + 1;
      else hi = mid;
    }
    const int j = lo - 1;
    double p, r;
    if (j < 0) {
      r = 0.0;
      p = 1.0;
    } else {
      const double rj = recall_of(tpc[j], nl), pj = __ddiv_rn((double)tpc[j], (double)(j + 1));
      const double xj = -(double)conf_of_key(keys[j]);
      if (j == n - 1 || xj == x) {
        r = rj;
        p = pj;
      } else {
        const double rj1 = recall_of(tpc[j + 1], nl), pj1 = __ddiv_rn((double)tpc[j + 1], (double)(j + 2));
        const double dx = __dsub_rn(-(double)conf_of_key(keys[j + 1]), xj), u = __dsub_rn(x, xj);
        r = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(rj1, rj), dx), u), rj);
        p = __dadd_rn(__dmul_rn(__ddiv_rn(__dsub_rn(pj1, pj), dx), u), pj);
      }
    }
    P[m] = p;
    R[m] = r;
    F[m] = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, p), r), __dadd_rn(__dadd_rn(p, r), 1e-16));
  }
}

// ------------------------------------------------------------------------------------------------
// summary (evaler.py:197-226): i* = last arg-max of f1.mean(0); mp, mr at i*; map50 = ap[:, 0].mean(); map = ap.mean(1).mean()
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) pr_summary_kernel(PrMetricArgs a) {
  const int nc = a.st.nc, tid = threadIdx.x;
  const double* P = a.out;
  const double* R = P + (int64_t)nc * kPrCurve;
  const double* F = R + (int64_t)nc * kPrCurve;
  const double* ap = F + (int64_t)nc * kPrCurve;
  double* nt = const_cast<double*>(ap) + nc * kPrNiou;
  double* mat = nt + nc;
  double* sum = mat + (nc + 1) * (nc + 1);
  __shared__ double s_v[32];
  __shared__ int s_i[32];
  for (int c = tid; c < nc; c += blockDim.x) nt[c] = (double)a.st.nt[c];
  if (a.st.confusion)
    for (int k = tid; k < (nc + 1) * (nc + 1); k += blockDim.x) mat[k] = (double)a.st.matrix[k];
  int ncu = 0;
  for (int c = 0; c < nc; ++c) ncu += a.st.nt[c] > 0;
  // f1.mean(0): classes added in order (numpy reduces axis 0 row by row), then one division; ties -> the last index
  double best = -1.0;
  int bi = -1;
  if (ncu > 0 && tid < kPrCurve) {
    double s = 0.0;
    bool first = true;
    for (int c = 0; c < nc; ++c) {
      if (a.st.nt[c] == 0) continue;
      s = first ? F[(int64_t)c * kPrCurve + tid] : __dadd_rn(s, F[(int64_t)c * kPrCurve + tid]);
      first = false;
    }
    best = __ddiv_rn(s, (double)ncu);
    bi = tid;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double v = __shfl_down_sync(0xffffffffu, best, o);
    const int i = __shfl_down_sync(0xffffffffu, bi, o);
    if (v > best || (v == best && i > bi)) best = v, bi = i;
  }
  if ((tid & 31) == 0) s_v[tid >> 5] = best, s_i[tid >> 5] = bi;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (s_v[w] > best || (s_v[w] == best && s_i[w] > bi)) best = s_v[w], bi = s_i[w];
    const bool ok = a.st.flags[1] != 0 && ncu > 0;          // stats[0].any(), else "Calculate metric failed"
    double mp = 0.0, mr = 0.0, map50 = 0.0, map = 0.0;
    if (ok) {
      for (int c = 0; c < nc; ++c) {
        if (a.st.nt[c] == 0) continue;
        mp = __dadd_rn(mp, P[(int64_t)c * kPrCurve + bi]);
        mr = __dadd_rn(mr, R[(int64_t)c * kPrCurve + bi]);
        map50 = __dadd_rn(map50, ap[c * kPrNiou]);
        double row = 0.0;
        for (int t = 0; t < kPrNiou; ++t) row = __dadd_rn(row, ap[c * kPrNiou + t]);
        map = __dadd_rn(map, __ddiv_rn(row, (double)kPrNiou));
      }
      const double d = (double)ncu;
      mp = __ddiv_rn(mp, d), mr = __ddiv_rn(mr, d), map50 = __ddiv_rn(map50, d), map = __ddiv_rn(map, d);
    }
    sum[0] = map50;
    sum[1] = map;
    sum[2] = mp;
    sum[3] = mr;
    sum[4] = ok ? (double)bi : -1.0;
    sum[5] = ok ? 1.0 : 0.0;
    sum[6] = (double)a.st.flags[0];
    sum[7] = (double)ncu;
  }
}

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

struct PrWs {
  uint64_t *ka, *kb;
  uint32_t *va, *vb, *hist;
  int32_t* tpc0;
};

static int64_t pr_layout(int64_t N, PrWs* w, char* base) {
  int64_t off = 0;
  auto take = [&](int64_t bytes) { const int64_t o = off; off += align256(bytes); return base ? base + o : (char*)nullptr; };
  w->ka = (uint64_t*)take(N * 8);
  w->kb = (uint64_t*)take(N * 8);
  w->va = (uint32_t*)take(N * 4);
  w->vb = (uint32_t*)take(N * 4);
  w->hist = (uint32_t*)take(rs_hist_words(N) * 4);
  w->tpc0 = (int32_t*)take(N * 4);
  return off;
}

static bool pr_state_ok(const yv6_pr_state* st) {
  return st && st->max_images > 0 && st->max_det > 0 && st->nc > 0 && st->conf && st->cls && st->correct && st->ndet && st->nt &&
         st->npred && st->flags && (!st->confusion || st->matrix);
}

}  // namespace yv6

using namespace yv6;

extern "C" int64_t yv6_pr_workspace_bytes(int32_t max_images, int32_t max_det) {
  PrWs w;
  return pr_layout((int64_t)std::max(max_images, 0) * std::max(max_det, 0), &w, nullptr);
}

extern "C" int yv6_pr_match(yv6_handle* h, const yv6_pr_state* st, const float* det, const int32_t* count, int32_t B, int32_t max_det,
                            const float* targets, int32_t n_targets, const float* meta, int32_t H, int32_t W, const float* iouv,
                            int32_t first_image, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && pr_state_ok(st) && det && count && meta && iouv, "pr_match: null argument or bad state");
  YV6_REQUIRE(B > 0 && B <= 65535 && max_det > 0 && max_det <= st->max_det, "pr_match: B=%d max_det=%d (state max_det %d)", B, max_det,
              st->max_det);
  YV6_REQUIRE(n_targets >= 0 && (n_targets == 0 || targets), "pr_match: bad targets");
  YV6_REQUIRE(H > 0 && W > 0, "pr_match: bad canvas %dx%d", H, W);
  YV6_REQUIRE(first_image >= 0 && (int64_t)first_image + B <= st->max_images, "pr_match: images %d..%d exceed max_images %d",
              first_image, first_image + B, st->max_images);
  const int64_t avail = (int64_t)h->max_smem_optin - 1024;          // opt-in limit less the kernel's static shared memory
  const int64_t det_bytes = (int64_t)max_det * 40;                   // dbox 16 + dconf, dcls, cm, dl, dmask, cl 4 each
  YV6_REQUIRE(det_bytes + 24 * 64 <= avail, "pr_match: max_det %d too large", max_det);
  const int lcap = (int)std::min<int64_t>(std::max(n_targets, 1), (avail - det_bytes) / 24);
  const size_t smem = (size_t)det_bytes + (size_t)lcap * 24;
  if (!(h->configured & YV6_CFG_METRICS)) {
    YV6_CHECK_CUDA(cudaFuncSetAttribute(pr_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)avail));
    h->configured |= YV6_CFG_METRICS;
  }
  PrMatchArgs a;
  a.st = *st;
  a.det = det;
  a.count = count;
  a.targets = targets;
  a.meta = meta;
  a.iouv = iouv;
  a.D = max_det;
  a.n = n_targets;
  a.H = H;
  a.W = W;
  a.first = first_image;
  a.lcap = lcap;
  pr_match_kernel<<<B, kMatchThreads, smem, (cudaStream_t)stream>>>(a);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_pr_metric(yv6_handle* h, const yv6_pr_state* st, int32_t n_images, const double* px, const double* x101,
                             void* workspace, int64_t workspace_bytes, double* out, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && pr_state_ok(st) && px && x101 && out, "pr_metric: null argument or bad state");
  YV6_REQUIRE(n_images >= 0 && n_images <= st->max_images, "pr_metric: n_images %d out of range", n_images);
  const int64_t N = (int64_t)n_images * st->max_det;
  YV6_REQUIRE(N < (1ll << 31), "pr_metric: %lld rows exceed the 32-bit slot index", (long long)N);
  PrWs w;
  const int64_t need = pr_layout(N, &w, reinterpret_cast<char*>(workspace));
  YV6_REQUIRE(N == 0 || (workspace && workspace_bytes >= need), "pr_metric: workspace too small (%lld < %lld)", (long long)workspace_bytes,
              (long long)need);
  cudaStream_t s = (cudaStream_t)stream;
  const int nc = st->nc;
  YV6_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * YV6_PR_OUT_SIZE(nc), s));
  PrMetricArgs a;
  a.st = *st;
  a.keys = w.ka;
  a.vals = w.va;
  a.tpc0 = w.tpc0;
  a.px = px;
  a.x101 = x101;
  a.out = out;
  if (N > 0) {
    pr_keys_kernel<<<(unsigned)((N + 255) / 256), 256, 0, s>>>(*st, N, w.ka, w.va);
    uint64_t *kin = w.ka, *kout = w.kb;
    uint32_t *vin = w.va, *vout = w.vb;
    for (int shift = 0; shift < 32 || (shift < 64 && ((uint64_t)nc >> (shift - 32)) != 0); shift += 8) {
      rs_pass(kin, vin, kout, vout, N, shift, w.hist, s);
      std::swap(kin, kout);
      std::swap(vin, vout);
    }
    a.keys = kin;
    a.vals = vin;
    pr_ap_kernel<<<dim3(nc, kPrNiou), kApThreads, 0, s>>>(a);
    pr_curve_kernel<<<nc, 256, 0, s>>>(a);
  }
  pr_summary_kernel<<<1, 1024, 0, s>>>(a);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
