// yv6_cocoeval.cu -- pycocotools' COCO box evaluation (COCOeval, iouType 'bbox', default Params) on the device, as the
// reference's Evaler.eval_model drives it (yolov6/core/evaler.py:231-321).
//
//   coco_match_kernel : one CTA per image of a batch.  The image's rows as pycocotools reads them back from the Evaler's
//                       predictions.json (yv6_eval_boxes' geometry, then round(v, 3) / round(v, 5) and a json round trip,
//                       restated as rint(v * 1e3) / 1e3 in double), or result rows given as doubles; per (image, category)
//                       the stable descending-score rank (the first 100 kept), and evaluateImg's greedy match against the
//                       pair's gts for each of the 4 area ranges x 10 IoU thresholds: one thread per (pair, range,
//                       threshold), IoU (maskApi.c bbIou) recomputed on the fly.  Outcomes land in a fixed slot per
//                       (image, row): two bits per (range, threshold), tp and fp (neither: the detection is ignored).
//   accumulate        : COCOeval.accumulate over every slot.  A stable LSD radix sort (yv6_sort.cuh) by descending score,
//                       then by category, reproduces the per-category np.argsort(-dtScores, kind='mergesort') over the
//                       per-image concatenation (slot order is sorted-imgId order; within an image and category, row order
//                       is rank order among equal scores).  One CTA per (category, range, maxDet, threshold) runs the
//                       cumulative tp / fp counts over the detections of rank < maxDet, the reverse running max of the
//                       precision and the 101 searchsorted queries.
//
// Every float64 operation that reaches an output or a comparison is an explicit round-to-nearest intrinsic in
// pycocotools' operation order (no FMA contraction: `(da + ga) - i` is the pattern nvcc would otherwise fuse), so
// precision / recall / scores are bit-identical to pycocotools'.  Thresholds and area ranges come from the host.
#include <algorithm>
#include <climits>

#include "yv6_common.cuh"
#include "yv6_handle.h"
#include "yv6_scale_coords.cuh"
#include "yv6_sort.cuh"

namespace yv6 {

constexpr int kCocoT = 10, kCocoR = 101, kCocoA = 4, kCocoM = 3;
constexpr int kCocoMaxDet = 100;                  // Params.maxDets[-1]: detections kept per (image, category)
constexpr int kMatchThreads = 256;
constexpr int kAccThreads = 256, kAccItems = 8, kAccChunk = kAccThreads * kAccItems;
constexpr int kRowBytes = 6 * 8 + 2 * 8 + 4 * 4;  // x, y, w, h, area, score; tp, fp; cat, rank, order, leader
enum { kCocoErrDetCls = 1 };

// Python's round(v, 3) of an fp32 value and the json round trip: v * 1e3 is exact in double (24 + 10 bits), rint rounds
// half to even like round(), and the division is correctly rounded
__device__ __forceinline__ double round_dec(float v, double scale) { return __ddiv_rn(rint(__dmul_rn((double)v, scale)), scale); }

// maskApi.c bbIou for one (dt, gt) pair of (x, y, w, h) boxes
__device__ __forceinline__ double bb_iou(double dx, double dy, double dw, double dh, const double* __restrict__ g, bool crowd) {
  const double gx = g[0], gy = g[1], gw = g[2], gh = g[3];
  const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(gw, gx)), fmax(dx, gx));
  if (w <= 0.0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(gh, gy)), fmax(dy, gy));
  if (h <= 0.0) return 0.0;
  const double i = __dmul_rn(w, h), da = __dmul_rn(dw, dh);
  const double u = crowd ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(gw, gh)), i);
  return __ddiv_rn(i, u);
}

// ------------------------------------------------------------------------------------------------
// per-image rows, ranks and greedy matching
// ------------------------------------------------------------------------------------------------
struct CocoMatchArgs {
  yv6_coco_state st;
  const float* det;        // MODE 0: [B][D][6] letterboxed xyxy, conf, cls
  const int32_t* count;    // MODE 0: [B]
  const float* meta;       // MODE 0: [B][6]
  const int32_t* cls_cat;  // MODE 0: [n_cls]
  const double* rows;      // MODE 1: [n][6] x, y, w, h, score, category index
  const int32_t* row_off;  // MODE 1: [B + 1]
  const int32_t* slots;    // [B]
  int32_t D, n_cls, W;     // rows per image held in shared memory, classes, matched-bit words per thread
};

template <int MODE>
__global__ void __launch_bounds__(kMatchThreads) coco_match_kernel(CocoMatchArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x, tid = threadIdx.x, D = a.D;
  const int slot = a.slots[b];
  if (slot < 0) return;                                     // an image outside params.imgIds
  double* sx = reinterpret_cast<double*>(smem);
  double *sy = sx + D, *sw = sy + D, *sh = sw + D, *sarea = sh + D, *sscore = sarea + D;
  unsigned long long* stp = reinterpret_cast<unsigned long long*>(sscore + D);
  unsigned long long* sfp = stp + D;
  int* scat = reinterpret_cast<int*>(sfp + D);
  int *srank = scat + D, *sorder = srank + D, *slead = sorder + D;
  uint32_t* mine = reinterpret_cast<uint32_t*>(slead + D) + tid * a.W;   // this thread's matched gts
  __shared__ double s_rng[2 * kCocoA], s_thr[kCocoT];
  __shared__ int s_nk, s_nl;
  const yv6_coco_state& st = a.st;

  const int n = MODE == 0 ? min(max(a.count[b], 0), D) : min(a.row_off[b + 1] - a.row_off[b], D);
  if (tid < 2 * kCocoA) s_rng[tid] = st.area_rng[tid];
  if (tid < kCocoT) s_thr[tid] = st.iou_thrs[tid];
  if (tid == 0) s_nk = s_nl = 0;
  const int64_t base = (int64_t)slot * st.max_det;
  for (int j = tid; j < n; j += kMatchThreads) {
    double x, y, w, h, s;
    int c;
    if (MODE == 0) {
      const float* r = a.det + ((int64_t)b * D + j) * 6;
      const float4 v = coco_xywh_rn(scale_coords_rn(r[0], r[1], r[2], r[3], a.meta + b * 6));
      x = round_dec(v.x, 1e3), y = round_dec(v.y, 1e3), w = round_dec(v.z, 1e3), h = round_dec(v.w, 1e3);
      s = round_dec(r[4], 1e5);
      const float cf = r[5];
      if (cf >= 0.f && cf < (float)a.n_cls && cf == floorf(cf)) {
        c = a.cls_cat[(int)cf];
      } else {
        c = -1;
        atomicOr(st.flags, kCocoErrDetCls);
      }
    } else {
      const double* r = a.rows + ((int64_t)a.row_off[b] + j) * 6;
      x = r[0], y = r[1], w = r[2], h = r[3], s = r[4];
      c = (int)r[5];
    }
    sx[j] = x, sy[j] = y, sw[j] = w, sh[j] = h;
    sarea[j] = __dmul_rn(w, h);                             // loadRes: area = bb[2] * bb[3]
    sscore[j] = s;
    scat[j] = c;
    st.score[base + j] = s;
    st.cat[base + j] = c;
  }
  __syncthreads();
  // rank in the (image, category) pair: np.argsort(-score, kind='mergesort'), ties in row (= result) order
  for (int j = tid; j < n; j += kMatchThreads) {
    const int c = scat[j];
    int r = INT_MAX;
    if (c >= 0) {
      const double s = sscore[j];
      r = 0;
      for (int i = 0; i < n; ++i) r += scat[i] == c && (sscore[i] > s || (sscore[i] == s && i < j));
    }
    srank[j] = r;
    stp[j] = sfp[j] = 0ull;
  }
  __syncthreads();
  // the kept detections in (category, rank) order: each pair is a contiguous run led by its rank-0 detection
  for (int j = tid; j < n; j += kMatchThreads) {
    const int c = scat[j], r = srank[j];
    const bool kept = c >= 0 && r < kCocoMaxDet;
    if (kept) {
      int p = 0;
      for (int i = 0; i < n; ++i) {
        const int ci = scat[i], ri = srank[i];
        p += ci >= 0 && ri < kCocoMaxDet && (ci < c || (ci == c && ri < r));
      }
      sorder[p] = j;
      atomicAdd(&s_nk, 1);
      if (r == 0) slead[atomicAdd(&s_nl, 1)] = p;
    }
    st.rank[base + j] = kept ? (uint8_t)r : (uint8_t)255;
  }
  __syncthreads();
  const int nk = s_nk, nl = s_nl, K = st.n_cats;
  // evaluateImg's greedy match, one thread per (pair, area range, threshold); the leader order does not matter, every
  // work item writes its own bit
  for (int it = tid; it < nl * kCocoA * kCocoT; it += kMatchThreads) {
    const int p0 = slead[it / (kCocoA * kCocoT)], at = it % (kCocoA * kCocoT), ar = at / kCocoT, t = at % kCocoT;
    const int c = scat[sorder[p0]];
    int len = 1;
    while (p0 + len < nk && scat[sorder[p0 + len]] == c) ++len;
    const int g0 = st.gt_off[(int64_t)slot * K + c], G = st.gt_off[(int64_t)slot * K + c + 1] - g0;
    for (int w = 0; w < a.W; ++w) mine[w] = 0u;
    const double lo = s_rng[2 * ar], hi = s_rng[2 * ar + 1];
    const double thr = fmin(s_thr[t], 1.0 - 1e-10);
    const unsigned long long bit = 1ull << at;
    const uint8_t* gf = st.gt_flags + g0;
    const double* ga = st.gt_area + g0;
    const double* gb = st.gt_box + (int64_t)g0 * 4;
    for (int q = 0; q < len; ++q) {
      const int d = sorder[p0 + q];
      const double dx = sx[d], dy = sy[d], dw = sw[d], dh = sh[d];
      double best = thr;
      int m = -1;
      // gts stable-sorted with the non-ignored ones first; a match among those ends the search before the ignored ones
      for (int pass = 0; pass < 2 && m < 0; ++pass) {
        for (int g = 0; g < G; ++g) {
          const bool crowd = gf[g] & 1;
          const bool ig = crowd || ga[g] < lo || ga[g] > hi;
          if (ig != (pass == 1)) continue;
          if (!crowd && ((mine[g >> 5] >> (g & 31)) & 1u)) continue;   // matched already and not a crowd
          const double iou = bb_iou(dx, dy, dw, dh, gb + (int64_t)g * 4, crowd);
          if (iou < best) continue;
          best = iou;
          m = g;
        }
      }
      bool dig = false, nz = false;                         // dtIg, dtm != 0
      if (m >= 0) {
        dig = (gf[m] & 1) || ga[m] < lo || ga[m] > hi;
        nz = (gf[m] & 2) != 0;                              // dtm holds the gt's id: id 0 reads as no match
        mine[m >> 5] |= 1u << (m & 31);
      }
      if (!nz) dig = dig || sarea[d] < lo || sarea[d] > hi;
      if (!dig) atomicOr(nz ? &stp[d] : &sfp[d], bit);
    }
  }
  __syncthreads();
  for (int j = tid; j < n; j += kMatchThreads) {
    st.tp[base + j] = stp[j];
    st.fp[base + j] = sfp[j];
  }
  if (tid == 0) st.ndet[slot] = n;
}

// ------------------------------------------------------------------------------------------------
// accumulate: sort keys, the sorted detections, per (category, range, maxDet, threshold) curves
// ------------------------------------------------------------------------------------------------
// descending order of a double as an ascending uint64 (-0.0 ties with 0.0, as in np.argsort)
__device__ __forceinline__ uint64_t score_desc_bits(double s) {
  const uint64_t u = s == 0.0 ? 0ull : (uint64_t)__double_as_longlong(s);
  return ~((u >> 63) ? ~u : (u | 0x8000000000000000ull));
}

__device__ __forceinline__ bool kept_det(const yv6_coco_state& st, int64_t s) {
  const int slot = (int)(s / st.max_det), j = (int)(s - (int64_t)slot * st.max_det);
  return j < st.ndet[slot] && st.cat[s] >= 0 && st.rank[s] < kCocoMaxDet;
}

__global__ void coco_keys_kernel(yv6_coco_state st, int64_t N, uint64_t* keys, uint32_t* vals, uint32_t* ckey, int32_t* cnt) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  const bool kept = kept_det(st, s);
  keys[s] = kept ? score_desc_bits(st.score[s]) : 0ull;
  ckey[s] = kept ? (uint32_t)st.cat[s] : (uint32_t)st.n_cats;  // dropped slots sort after every category
  vals[s] = (uint32_t)s;
  if (kept) atomicAdd(cnt + st.cat[s], 1);
}

__global__ void coco_cat_keys_kernel(int64_t N, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ ckey, uint64_t* keys) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) keys[i] = ckey[vals[i]];
}

struct CocoSorted {
  double* score;
  uint64_t *tp, *fp;
  uint8_t* rank;
};

__global__ void coco_gather_kernel(yv6_coco_state st, int64_t N, const uint32_t* __restrict__ vals, CocoSorted o) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const uint32_t v = vals[i];
  o.score[i] = st.score[v];
  o.tp[i] = st.tp[v];
  o.fp[i] = st.fp[v];
  o.rank[i] = st.rank[v];
}

struct CocoAccArgs {
  yv6_coco_state st;
  CocoSorted srt;
  const int32_t* cnt;      // [K] kept detections per category
  double *precision, *recall, *scores;
};

__global__ void __launch_bounds__(kAccThreads) coco_accum_kernel(CocoAccArgs a) {
  const int k = blockIdx.x, y = blockIdx.y, tid = threadIdx.x;
  const int t = y / (kCocoA * kCocoM), ar = (y / kCocoM) % kCocoA, mi = y % kCocoM;
  const int K = a.st.n_cats, max_det = mi == 0 ? 1 : (mi == 1 ? 10 : 100);   // Params.maxDets
  const int bit = ar * kCocoT + t;
  const int64_t col = (int64_t)k * kCocoA * kCocoM + ar * kCocoM + mi, rstride = (int64_t)K * kCocoA * kCocoM;
  double* prec = a.precision + (int64_t)t * kCocoR * rstride + col;
  double* scs = a.scores + (int64_t)t * kCocoR * rstride + col;
  double* rec = a.recall + (int64_t)t * rstride + col;
  const int npig = a.st.npig[k * kCocoA + ar];
  if (npig == 0) {                                          // no gt that counts: pycocotools leaves -1
    for (int r = tid; r < kCocoR; r += kAccThreads) prec[r * rstride] = scs[r * rstride] = -1.0;
    if (tid == 0) *rec = -1.0;
    return;
  }
  int start = 0;
  for (int c = 0; c < k; ++c) start += a.cnt[c];
  const int n = a.cnt[k];
  const double* score = a.srt.score + start;
  const uint64_t* tpm = a.srt.tp + start;
  const uint64_t* fpm = a.srt.fp + start;
  const uint8_t* rank = a.srt.rank + start;
  __shared__ int s_K[kCocoR], s_P[kCocoR], s_wi[32], s_first;
  __shared__ double s_env[kCocoR], s_wd[32], s_chunk[kAccChunk];
  if (tid < kCocoR) {
    // searchsorted(rc, recThrs[r], 'left') is the first detection whose running tp count reaches K = the least c with
    // c / npig >= recThrs[r]
    const double x = a.st.rec_thrs[tid];
    int c = min(max((int)(x * npig) - 1, 0), npig);
    while (c > 0 && __ddiv_rn((double)(c - 1), (double)npig) >= x) --c;
    while (c <= npig && __ddiv_rn((double)c, (double)npig) < x) ++c;
    s_K[tid] = c;
    s_P[tid] = -1;
    s_env[tid] = 0.0;
  }
  if (tid == 0) s_first = INT_MAX;
  __syncthreads();
  // forward: running tp counts over the detections of rank < maxDet; the position of each query's K-th tp
  int T = 0, TF = 0, nd = 0;
  for (int cb = 0; cb < n; cb += kAccChunk) {
    const int i0 = cb + tid * kAccItems;
    int tbits = 0, ntp = 0, nfp = 0, nf = 0, first = INT_MAX;
#pragma unroll
    for (int q = 0; q < kAccItems; ++q) {
      const int i = i0 + q;
      const bool f = i < n && rank[i] < max_det;
      const int tp = f ? (int)((tpm[i] >> bit) & 1ull) : 0;
      tbits |= tp << q;
      ntp += tp;
      nfp += f ? (int)((fpm[i] >> bit) & 1ull) : 0;
      nf += f;
      if (f) first = min(first, i);
    }
    if (first != INT_MAX) atomicMin(&s_first, first);
    int tot, totf, totfp;
    int tpc = T + block_excl_sum(ntp, s_wi, &tot);
#pragma unroll
    for (int q = 0; q < kAccItems; ++q) {
      if (!((tbits >> q) & 1)) continue;
      ++tpc;
      int lo = 0, hi = kCocoR;                              // first query with K >= tpc
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_K[mid] < tpc) lo = mid + 1;
        else hi = mid;
      }
      for (int r = lo; r < kCocoR && s_K[r] == tpc; ++r) s_P[r] = i0 + q;
    }
    block_excl_sum(nf, s_wi, &totf);
    block_excl_sum(nfp, s_wi, &totfp);
    T += tot;
    nd += totf;
    TF += totfp;
  }
  __syncthreads();
  if (tid < kCocoR && s_K[tid] == 0 && nd > 0) s_P[tid] = s_first;
  // reverse: pr[i-1] = max(pr[i-1], pr[i]) from the end, read at the queries' positions
  int after_tp = 0, after_fp = 0;
  double cmax = 0.0;
  const int nchunks = (n + kAccChunk - 1) / kAccChunk;
  for (int ci = nchunks - 1; ci >= 0; --ci) {
    const int cb = ci * kAccChunk, i0 = cb + tid * kAccItems;
    int fbits = 0, tbits = 0, pbits = 0, ntp = 0, nfp = 0;
#pragma unroll
    for (int q = 0; q < kAccItems; ++q) {
      const int i = i0 + q;
      const bool f = i < n && rank[i] < max_det;
      const int tp = f ? (int)((tpm[i] >> bit) & 1ull) : 0, fp = f ? (int)((fpm[i] >> bit) & 1ull) : 0;
      fbits |= (int)f << q;
      tbits |= tp << q;
      pbits |= fp << q;
      ntp += tp;
      nfp += fp;
    }
    int tot_tp, tot_fp;
    const int ex_tp = block_excl_sum(ntp, s_wi, &tot_tp);
    const int ex_fp = block_excl_sum(nfp, s_wi, &tot_fp);
    int tpc = T - after_tp - tot_tp + ex_tp, fpc = TF - after_fp - tot_fp + ex_fp;
    double pr[kAccItems];
    double tmax = 0.0;
#pragma unroll
    for (int q = 0; q < kAccItems; ++q) {
      tpc += (tbits >> q) & 1;
      fpc += (pbits >> q) & 1;
      // pr = tp / (fp + tp + np.spacing(1))
      pr[q] = ((fbits >> q) & 1) ? __ddiv_rn((double)tpc, __dadd_rn((double)(fpc + tpc), 2.220446049250313e-16)) : 0.0;
      tmax = fmax(tmax, pr[q]);
    }
    double ctot;
    double run = fmax(block_excl_sufmax(tmax, s_wd, &ctot), cmax);
#pragma unroll
    for (int q = kAccItems - 1; q >= 0; --q) {
      run = fmax(run, pr[q]);
      if (i0 + q < n) s_chunk[tid * kAccItems + q] = run;
    }
    __syncthreads();
    if (tid < kCocoR) {
      const int P = s_P[tid];
      if (P >= cb && P < cb + kAccChunk) s_env[tid] = s_chunk[P - cb];
    }
    after_tp += tot_tp;
    after_fp += tot_fp;
    cmax = fmax(cmax, ctot);
    __syncthreads();
  }
  if (tid < kCocoR) {
    const int P = s_P[tid];                                 // -1: searchsorted ran off the end, the entry stays 0
    prec[tid * rstride] = P >= 0 ? s_env[tid] : 0.0;
    scs[tid * rstride] = P >= 0 ? score[P] : 0.0;
  }
  if (tid == 0) *rec = nd > 0 ? __ddiv_rn((double)T, (double)npig) : 0.0;
}

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

struct CocoWs {
  uint64_t *ka, *kb;
  uint32_t *va, *vb, *ckey, *hist;
  int32_t* cnt;
  CocoSorted srt;
};

static int64_t coco_layout(int64_t N, int K, CocoWs* w, char* base) {
  int64_t off = 0;
  auto take = [&](int64_t bytes) { const int64_t o = off; off += align256(bytes); return base ? base + o : (char*)nullptr; };
  w->ka = (uint64_t*)take(N * 8);
  w->kb = (uint64_t*)take(N * 8);
  w->va = (uint32_t*)take(N * 4);
  w->vb = (uint32_t*)take(N * 4);
  w->ckey = (uint32_t*)take(N * 4);
  w->hist = (uint32_t*)take(rs_hist_words(N) * 4);
  w->cnt = (int32_t*)take((int64_t)K * 4);
  w->srt.score = (double*)take(N * 8);
  w->srt.tp = (uint64_t*)take(N * 8);
  w->srt.fp = (uint64_t*)take(N * 8);
  w->srt.rank = (uint8_t*)take(N);
  return off;
}

static bool coco_state_ok(const yv6_coco_state* st) {
  return st && st->n_images > 0 && st->n_cats > 0 && st->max_det > 0 && st->max_gts >= 0 && st->gt_off && st->npig && st->area_rng &&
         st->iou_thrs && st->rec_thrs && st->score && st->cat && st->rank && st->tp && st->fp && st->ndet && st->flags &&
         (int64_t)st->n_images * st->max_det < (1ll << 31);
}

template <int MODE>
static int coco_match_launch(yv6_handle* h, CocoMatchArgs& a, int B, cudaStream_t s) {
  a.W = std::max(1, (a.st.max_gts + 31) / 32);
  const int64_t avail = (int64_t)h->max_smem_optin - 1024;  // opt-in limit less the kernel's static shared memory
  const int64_t smem = (int64_t)a.D * kRowBytes + (int64_t)kMatchThreads * a.W * 4;
  YV6_REQUIRE(smem <= avail, "coco: %d rows per image and %d gts per (image, category) need %lld bytes of shared memory (> %lld)", a.D,
              a.st.max_gts, (long long)smem, (long long)avail);
  if (!(h->configured & YV6_CFG_COCO)) {
    YV6_CHECK_CUDA(cudaFuncSetAttribute(coco_match_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)avail));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(coco_match_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)avail));
    h->configured |= YV6_CFG_COCO;
  }
  coco_match_kernel<MODE><<<B, kMatchThreads, (size_t)smem, s>>>(a);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

}  // namespace yv6

using namespace yv6;

extern "C" int64_t yv6_coco_workspace_bytes(int32_t n_images, int32_t max_det, int32_t n_cats) {
  CocoWs w;
  return coco_layout((int64_t)std::max(n_images, 0) * std::max(max_det, 0), std::max(n_cats, 0), &w, nullptr);
}

extern "C" int yv6_coco_update(yv6_handle* h, const yv6_coco_state* st, const float* det, const int32_t* count, const float* meta,
                               const int32_t* cls_cat, int32_t n_cls, const int32_t* slots, int32_t B, int32_t max_det, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && coco_state_ok(st) && det && count && meta && cls_cat && slots, "coco_update: null argument or bad state");
  YV6_REQUIRE(B > 0 && B <= 65535 && max_det > 0 && max_det <= st->max_det && n_cls > 0, "coco_update: B=%d max_det=%d (state %d) n_cls=%d",
              B, max_det, st->max_det, n_cls);
  CocoMatchArgs a{};
  a.st = *st;
  a.det = det;
  a.count = count;
  a.meta = meta;
  a.cls_cat = cls_cat;
  a.slots = slots;
  a.D = max_det;
  a.n_cls = n_cls;
  return coco_match_launch<0>(h, a, B, (cudaStream_t)stream);
}

extern "C" int yv6_coco_load(yv6_handle* h, const yv6_coco_state* st, const double* rows, const int32_t* row_off, const int32_t* slots,
                             int32_t B, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && coco_state_ok(st) && rows && row_off && slots, "coco_load: null argument or bad state");
  YV6_REQUIRE(B > 0 && B <= 65535, "coco_load: B=%d", B);
  CocoMatchArgs a{};
  a.st = *st;
  a.rows = rows;
  a.row_off = row_off;
  a.slots = slots;
  a.D = st->max_det;
  return coco_match_launch<1>(h, a, B, (cudaStream_t)stream);
}

extern "C" int yv6_coco_accumulate(yv6_handle* h, const yv6_coco_state* st, void* workspace, int64_t workspace_bytes, double* precision,
                                   double* recall, double* scores, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && coco_state_ok(st) && workspace && precision && recall && scores, "coco_accumulate: null argument or bad state");
  YV6_REQUIRE(st->n_cats <= 65535, "coco_accumulate: %d categories exceed the grid", st->n_cats);
  const int64_t N = (int64_t)st->n_images * st->max_det;
  const int K = st->n_cats;
  CocoWs w;
  const int64_t need = coco_layout(N, K, &w, reinterpret_cast<char*>(workspace));
  YV6_REQUIRE(workspace_bytes >= need, "coco_accumulate: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
  cudaStream_t s = (cudaStream_t)stream;
  YV6_CHECK_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * K, s));
  const unsigned nb = (unsigned)((N + 255) / 256);
  coco_keys_kernel<<<nb, 256, 0, s>>>(*st, N, w.ka, w.va, w.ckey, w.cnt);
  uint64_t *kin = w.ka, *kout = w.kb;
  uint32_t *vin = w.va, *vout = w.vb;
  for (int shift = 0; shift < 64; shift += 8) {             // descending score, all 64 bits: the row path takes any double
    rs_pass(kin, vin, kout, vout, N, shift, w.hist, s);
    std::swap(kin, kout);
    std::swap(vin, vout);
  }
  coco_cat_keys_kernel<<<nb, 256, 0, s>>>(N, vin, w.ckey, kin);
  for (int shift = 0; shift == 0 || (K >> shift) != 0; shift += 8) {   // then category (K = dropped slots)
    rs_pass(kin, vin, kout, vout, N, shift, w.hist, s);
    std::swap(kin, kout);
    std::swap(vin, vout);
  }
  coco_gather_kernel<<<nb, 256, 0, s>>>(*st, N, vin, w.srt);
  CocoAccArgs a;
  a.st = *st;
  a.srt = w.srt;
  a.cnt = w.cnt;
  a.precision = precision;
  a.recall = recall;
  a.scores = scores;
  coco_accum_kernel<<<dim3(K, kCocoT * kCocoA * kCocoM), kAccThreads, 0, s>>>(a);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
