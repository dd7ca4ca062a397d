// yv6_nms.cu -- batched non-maximum suppression for all images of a batch in three launches.
//
// Reference: `non_max_suppression` (yolov6/utils/nms.py:31-105) which loops over images in Python,
// compacts with boolean masks and calls torchvision.ops.nms per image (nms.py:96).  Here:
//   1. nms_select : one warp-per-anchor-row pass over pred[B,A,5+nc] (coalesced class reads, pred is read
//                   exactly once): candidate rule of nms.py:48, obj*cls (nms.py:69), best class
//                   (nms.py:79-80) or every class above the threshold (nms.py:75-77); survivors take a
//                   slot from a per-image atomic counter and write box (xywh->xyxy, nms.py:21-28),
//                   score, class, anchor and a 64-bit key (descending score, ascending anchor*nc+class).
//   2. nms_sort   : one block per image, bitonic key-value sort (value = slot).  The key order is a total
//                   order equal to torchvision's stable descending sort over the reference's candidate
//                   list, whose order is anchor-major / class-minor (`nonzero`, nms.py:76).
//   3. nms_greedy : one block per image, greedy suppression in chunks of 64 sorted candidates against
//                   the kept set; class offset boxes + cls*4096 (nms.py:94-95); float IoU promoted to
//                   double against the double threshold exactly like torchvision's CPU kernel; stops
//                   at max_det (nms.py:97-98); at most max_nms = 30000 candidates enter (nms.py:90-91).
// All fp32 arithmetic that feeds a comparison uses explicit round-to-nearest intrinsics (no FMA
// contraction) in the reference's operation order, so kept indices and class ids are bit-exact.
#include <algorithm>

#include "yv6_common.cuh"
#include "yv6_handle.h"
#include "yv6_scale_coords.cuh"

namespace yv6 {

constexpr int kNmsTile = 256;       // anchors per block in scan/emit
constexpr int kMaxNms = 30000;      // nms.py:55
constexpr int kMultiCap = 65536;    // candidate capacity per image in multi-label mode
constexpr int kSortSmemMax = 16384; // keys sorted in shared memory up to this many
constexpr int kTopK = 2048;         // size the sorted prefix aims at
constexpr int kTopCap = 8192;       // ... and may reach (one histogram bin can hold many keys); beyond it the full sort runs
constexpr int kHistBins = 4096;     // overflow pre-selection: bins over bits [30:19] of the (positive) fp32 score

__device__ __forceinline__ float4 xywh2xyxy_rn(float x, float y, float w, float h) {
  const float hw = __fdiv_rn(w, 2.f), hh = __fdiv_rn(h, 2.f);               // nms.py:24-27
  return make_float4(__fsub_rn(x, hw), __fsub_rn(y, hh), __fadd_rn(x, hw), __fadd_rn(y, hh));
}

struct NmsWs {
  int32_t* cand_count;   // [B] slots taken (may exceed cap; clamped by the consumers)
  int32_t* overflow;     // [1]
  uint64_t* keys;        // [B][cap2]
  uint32_t* hist;        // [B][kHistBins] score histogram of the images that overflowed `cap` (null when cap covers A*nc)
  int32_t* cutoff;       // [B] lowest histogram bin that still enters the sort, -1 = image did not overflow
  // top-K prefix (head mode): the greedy pass stops at max_det kept boxes and normally consumes only the best few hundred
  // candidates, so only the best ~kTopK keys of an image are sorted first; the full sort runs only if they did not suffice
  uint32_t* top_hist;    // [B][kHistBins] score histogram of every candidate (filled by nms_select_rows_kernel), or null
  uint64_t* top_keys;    // [B][kTopCap] sorted prefix
  int32_t* top_n;        // [B] keys in the prefix; -1 = the prefix IS the whole (fully sorted) list in `keys`
  int32_t* need_full;    // [B] set by the greedy pass when the prefix ran out before max_det boxes were kept
  int32_t cap, cap2, T;
};

constexpr int kNmsMaxLevels = 6;
struct NmsParams {
  // score rows: `rows` + (b*A + a) * row_pitch; class c at [cls_off + c]; objectness at [4] when has_obj, else 1.0
  //   pred mode: rows = pred [B,A,5+nc], row_pitch = 5+nc, cls_off = 5, has_obj = 1, boxes = rows[0..3] (xywh)
  //   head mode: rows = cls  [B,A,nc],   row_pitch = nc,   cls_off = 0, has_obj = 0, boxes decoded from `reg` on demand
  const float* rows;
  int32_t row_pitch, cls_off, has_obj;
  const float* reg;      // head mode: [B,A,R] ltrb distances or DFL logits
  int32_t R, reg_max, nl;
  int32_t lvl_off[kNmsMaxLevels + 1];
  int32_t lvl_w[kNmsMaxLevels];
  float lvl_stride[kNmsMaxLevels];
  int32_t B, A, nc, no;
  float conf;
  double iou;
  int32_t agnostic, multi_label, max_det;
  const uint8_t* class_mask;
  float* out;
  int32_t* out_count;
  int32_t* out_src;
  NmsWs ws;
};

// xyxy box of anchor `anchor` of image b.  Head mode repeats, operation for operation, what head_decode_kernel (yv6_aux.cu:
// effidehead.py:106-139, general.py:32-43) writes into `pred` and what the pred mode then reads back, so both modes keep the
// same rows bit for bit.
__device__ __forceinline__ float4 candidate_box(const NmsParams& p, int b, int anchor) {
  if (p.has_obj) {
    const float* r = p.rows + ((int64_t)b * p.A + anchor) * p.row_pitch;
    return xywh2xyxy_rn(__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3));
  }
  const float* reg = p.reg + ((int64_t)b * p.A + anchor) * p.R;
  float d[4];
  if (p.R == 4) {
#pragma unroll
    for (int k = 0; k < 4; ++k) d[k] = __ldg(reg + k);
  } else {
    const int nb = p.reg_max + 1;
    for (int k = 0; k < 4; ++k) {
      const float* l = reg + k * nb;
      float mx = -INFINITY;
      for (int i = 0; i < nb; ++i) mx = fmaxf(mx, __ldg(l + i));
      float den = 0.f;
      for (int i = 0; i < nb; ++i) den += expf(__ldg(l + i) - mx);
      float e = 0.f;
      for (int i = 0; i < nb; ++i) e = __fadd_rn(e, __fmul_rn(expf(__ldg(l + i) - mx) / den, (float)i));
      d[k] = e;
    }
  }
  int lvl = 0;
  while (lvl + 1 < p.nl && anchor >= p.lvl_off[lvl + 1]) ++lvl;
  const int local = anchor - p.lvl_off[lvl];
  const float ax = (float)(local % p.lvl_w[lvl]) + 0.5f;
  const float ay = (float)(local / p.lvl_w[lvl]) + 0.5f;
  const float st = p.lvl_stride[lvl];
  const float x1 = __fsub_rn(ax, d[0]), y1 = __fsub_rn(ay, d[1]);
  const float x2 = __fadd_rn(ax, d[2]), y2 = __fadd_rn(ay, d[3]);
  return xywh2xyxy_rn(__fmul_rn(__fdiv_rn(__fadd_rn(x1, x2), 2.f), st), __fmul_rn(__fdiv_rn(__fadd_rn(y1, y2), 2.f), st),
                      __fmul_rn(__fsub_rn(x2, x1), st), __fmul_rn(__fsub_rn(y2, y1), st));
}


__device__ __forceinline__ uint64_t make_key(float score, int order) {
  return ((uint64_t)(0xffffffffu - __float_as_uint(score)) << 32) | (uint32_t)order;  // score > 0
}

// Hits of anchor rows; lanes own classes lane, lane+32, ...  R rows are scanned together so that their loads
// and shuffle reductions overlap (the pass is latency-bound otherwise).  (nms.py:48,69,75-84)
struct RowScan {
  float obj, raw_max, best;
  int best_c, cnt;        // cnt: warp total of (score > conf and class allowed)
};
template <int R>
__device__ __forceinline__ void scan_rows(const NmsParams& p, const float* const (&row)[R], const bool (&ok)[R], int lane,
                                          RowScan (&r)[R]) {
#pragma unroll
  for (int q = 0; q < R; ++q) {
    r[q].obj = ok[q] ? (p.has_obj ? __ldg(row[q] + 4) : 1.f) : 0.f;
    r[q].raw_max = -INFINITY;
    r[q].best = -INFINITY;
    r[q].best_c = 0x7fffffff;
    r[q].cnt = 0;
  }
  for (int c = lane; c < p.nc; c += 32) {
    const bool cls_ok = (p.class_mask == nullptr) || (p.class_mask[c] != 0);
    float v[R];
#pragma unroll
    for (int q = 0; q < R; ++q) v[q] = ok[q] ? __ldg(row[q] + p.cls_off + c) : -INFINITY;
#pragma unroll
    for (int q = 0; q < R; ++q) {
      r[q].raw_max = fmaxf(r[q].raw_max, v[q]);
      const float s = __fmul_rn(v[q], r[q].obj);                           // nms.py:69
      if (s > r[q].best) { r[q].best = s; r[q].best_c = c; }               // first max within the lane
      if (s > p.conf && cls_ok) ++r[q].cnt;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int q = 0; q < R; ++q) {
      r[q].raw_max = fmaxf(r[q].raw_max, __shfl_xor_sync(0xffffffffu, r[q].raw_max, o));
      const float ob = __shfl_xor_sync(0xffffffffu, r[q].best, o);
      const int oc = __shfl_xor_sync(0xffffffffu, r[q].best_c, o);
      if (ob > r[q].best || (ob == r[q].best && oc < r[q].best_c)) { r[q].best = ob; r[q].best_c = oc; }  // first max overall
      r[q].cnt += __shfl_xor_sync(0xffffffffu, r[q].cnt, o);
    }
  }
}

__device__ __forceinline__ int row_entries(const NmsParams& p, const RowScan& r) {
  const bool cand = (r.obj > p.conf) && (r.raw_max > p.conf);              // nms.py:48
  if (p.multi_label) return cand ? r.cnt : 0;                              // nms.py:75-77
  const bool cls_ok = (p.class_mask == nullptr) || (r.best_c < p.nc && p.class_mask[r.best_c] != 0);
  return (cand && r.best > p.conf && cls_ok) ? 1 : 0;                      // nms.py:79-84
}

// One warp per 32 anchor rows.  Pass 1 counts the entries of each row (lane i keeps row i's count), one
// atomicAdd per warp reserves the key slots, pass 2 revisits only the rows that have entries (L1/L2 hits)
// and writes their keys.  Key = (descending score, ascending anchor*nc + class): everything the greedy
// pass needs (anchor, class, exact score) is encoded in it, the box is re-read from `pred`.
__global__ void __launch_bounds__(kNmsTile) nms_select_kernel(const NmsParams p) {
  constexpr int R = 4;
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t* keys = p.ws.keys + (int64_t)b * p.ws.cap2;
  const int a0 = blockIdx.x * kNmsTile + warp * 32;
  if (a0 >= p.A) return;
  const float* img = p.rows + (int64_t)b * p.A * p.row_pitch;
  int my_entries = 0;                                                      // lane i: entries of row a0 + i
  for (int i0 = 0; i0 < 32; i0 += R) {
    const float* row[R];
    bool ok[R];
    RowScan r[R];
#pragma unroll
    for (int q = 0; q < R; ++q) {
      ok[q] = (a0 + i0 + q < p.A);
      row[q] = img + (int64_t)(a0 + i0 + q) * p.row_pitch;
    }
    scan_rows<R>(p, row, ok, lane, r);
#pragma unroll
    for (int q = 0; q < R; ++q) {
      const int e = ok[q] ? row_entries(p, r[q]) : 0;
      if (lane == i0 + q) my_entries = e;
    }
  }
  int incl = my_entries;                                                   // inclusive prefix over the 32 rows
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  if (total == 0) return;
  int slot0 = 0;
  if (lane == 0) slot0 = atomicAdd(&p.ws.cand_count[b], total);
  slot0 = __shfl_sync(0xffffffffu, slot0, 0);
  const int row_slot = slot0 + incl - my_entries;
  if (!p.multi_label) {
    for (int i0 = 0; i0 < 32; i0 += R) {
      const float* row[R];
      bool ok[R];
      RowScan r[R];
      bool any = false;
#pragma unroll
      for (int q = 0; q < R; ++q) {
        ok[q] = __shfl_sync(0xffffffffu, my_entries, i0 + q) != 0;
        row[q] = img + (int64_t)(a0 + i0 + q) * p.row_pitch;
        any = any || ok[q];
      }
      if (!any) continue;  // warp-uniform
      scan_rows<R>(p, row, ok, lane, r);
#pragma unroll
      for (int q = 0; q < R; ++q) {
        const int slot = __shfl_sync(0xffffffffu, row_slot, i0 + q);
        if (ok[q] && lane == 0 && slot < p.ws.cap) keys[slot] = make_key(r[q].best, a0 + i0 + q);
      }
    }
    return;
  }
  for (int i0 = 0; i0 < 32; i0 += R) {
    bool ok[R];
    int slot[R];
    float obj[R];
    bool any = false;
#pragma unroll
    for (int q = 0; q < R; ++q) {
      ok[q] = __shfl_sync(0xffffffffu, my_entries, i0 + q) != 0;
      slot[q] = __shfl_sync(0xffffffffu, row_slot, i0 + q);
      any = any || ok[q];
    }
    if (!any) continue;  // warp-uniform
#pragma unroll
    for (int q = 0; q < R; ++q) obj[q] = ok[q] ? (p.has_obj ? __ldg(img + (int64_t)(a0 + i0 + q) * p.row_pitch + 4) : 1.f) : 0.f;
    for (int c0 = 0; c0 < p.nc; c0 += 32) {                               // class-ascending within each row
      const int c = c0 + lane;
      const bool cls_ok = (c < p.nc) && ((p.class_mask == nullptr) || (p.class_mask[c] != 0));
      float v[R];
#pragma unroll
      for (int q = 0; q < R; ++q) v[q] = (ok[q] && c < p.nc) ? __ldg(img + (int64_t)(a0 + i0 + q) * p.row_pitch + p.cls_off + c) : 0.f;
#pragma unroll
      for (int q = 0; q < R; ++q) {
        const float sv = __fmul_rn(v[q], obj[q]);
        const bool hit = ok[q] && cls_ok && (sv > p.conf);
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) {
          const int my = slot[q] + __popc(m & ((1u << lane) - 1u));
          if (my < p.ws.cap) keys[my] = make_key(sv, (a0 + i0 + q) * p.nc + c);
        }
        slot[q] += __popc(m);
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// More than `cap` multi-label candidates in one image (an under-trained model at the Evaler's conf 0.03):
// the reference keeps the 30000 best by confidence (nms.py:90-91).  The three kernels below do nothing for
// images that fit.  For an image that overflowed they (1) histogram the candidate scores over 4096 bins
// that are monotone in the score, (2) find the lowest bin such that the bins from it upwards hold at least
// max_nms candidates, (3) re-emit only the candidates of those bins.  The sort then orders them by the full
// key, so the first 30000 are exactly the 30000 best under the stable order.  Only if the kept bins still
// hold more than `cap` keys (tens of thousands of scores equal to 8 significant bits) is `overflow` raised.

// bins over bits [30:19] of a positive fp32 score: monotone in the score
__device__ __forceinline__ int score_bin(float s) { return (int)((__float_as_uint(s) >> 19) & (kHistBins - 1)); }

// ------------------------------------------------------------------------------------------------
// Candidate selection for the head-tensor mode (rows = cls [B,A,nc], contiguous, objectness 1): each warp stages 32
// consecutive rows (one contiguous 32*nc*4-byte chunk, 16-byte loads) in shared memory with an odd row pitch and every LANE
// then walks ONE row from shared memory -- no cross-lane reductions at all (the generic kernel above spends most of its
// instructions in shuffles: five rounds x four values per row).  Same candidate rule, same keys.
constexpr int kSelRows = 32;
__global__ void __launch_bounds__(256) nms_select_rows_kernel(const NmsParams p) {
  extern __shared__ float sel_smem[];                       // [8 warps][32 rows][pitch]
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pitch = p.nc | 1;                               // odd -> lane-per-row reads are bank-conflict free
  float* tile = sel_smem + (size_t)warp * kSelRows * pitch;
  const int a0 = (blockIdx.x * 8 + warp) * kSelRows;
  if (a0 >= p.A) return;
  const int nrows = min(kSelRows, p.A - a0);
  const float* src = p.rows + ((int64_t)b * p.A + a0) * p.nc;
  const int total = nrows * p.nc;                           // floats; row starts are 16-byte aligned (nc % 4 == 0)
  // Eight 16-byte loads per lane are issued before the first one is consumed: the staging loop is otherwise one exposed
  // DRAM round trip per 512 bytes of the warp (20 of them for 80 classes -- the kernel ran at 1.5 TB/s).
  constexpr int kBatch = 8;
  for (int i0 = lane * 4; i0 < total; i0 += 128 * kBatch) {
    float4 v[kBatch];
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int i = i0 + 128 * j;
      if (i < total) v[j] = __ldcs(reinterpret_cast<const float4*>(src + i));   // streamed once: evict-first
    }
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int i = i0 + 128 * j;
      if (i < total) {
        const int r = i / p.nc, c = i - r * p.nc;           // nc % 4 == 0: a float4 never straddles two rows
        float* d = tile + r * pitch + c;
        d[0] = v[j].x; d[1] = v[j].y; d[2] = v[j].z; d[3] = v[j].w;
      }
    }
  }
  __syncwarp();
  const bool ok = lane < nrows;
  const float* row = tile + lane * pitch;
  float raw_max = -INFINITY, best = -INFINITY;
  int best_c = 0, cnt = 0;
  if (ok) {
    for (int c = 0; c < p.nc; ++c) {
      const float v = row[c];                               // obj = 1: score = v * 1.0f = v (nms.py:69)
      raw_max = fmaxf(raw_max, v);
      if (v > best) { best = v; best_c = c; }               // first max (nms.py:79)
      const bool cls_ok = (p.class_mask == nullptr) || (p.class_mask[c] != 0);
      if (v > p.conf && cls_ok) ++cnt;
    }
  }
  const bool cand = ok && (1.f > p.conf) && (raw_max > p.conf);                 // nms.py:48
  int entries;
  if (p.multi_label) {
    entries = cand ? cnt : 0;                                                   // nms.py:75-77
  } else {
    const bool cls_ok = (p.class_mask == nullptr) || (p.class_mask[best_c] != 0);
    entries = (cand && best > p.conf && cls_ok) ? 1 : 0;                        // nms.py:79-84
  }
  int incl = entries;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const int tot = __shfl_sync(0xffffffffu, incl, 31);
  if (tot == 0) return;
  int slot0 = 0;
  if (lane == 0) slot0 = atomicAdd(&p.ws.cand_count[b], tot);
  slot0 = __shfl_sync(0xffffffffu, slot0, 0);
  int slot = slot0 + incl - entries;
  if (entries == 0) return;
  uint64_t* keys = p.ws.keys + (int64_t)b * p.ws.cap2;
  const int a = a0 + lane;
  uint32_t* th = p.ws.top_hist + (int64_t)b * kHistBins;
  if (!p.multi_label) {
    if (slot < p.ws.cap) keys[slot] = make_key(best, a);
    atomicAdd(&th[score_bin(best)], 1u);
    return;
  }
  for (int c = 0; c < p.nc; ++c) {                                              // class-ascending within the row
    const float v = row[c];
    const bool cls_ok = (p.class_mask == nullptr) || (p.class_mask[c] != 0);
    if (v > p.conf && cls_ok) {
      if (slot < p.ws.cap) keys[slot] = make_key(v, a * p.nc + c);
      atomicAdd(&th[score_bin(v)], 1u);
      ++slot;
    }
  }
}

constexpr int kOverflowRows = 64;
template <bool EMIT>
__device__ __forceinline__ void overflow_row(const NmsParams& p, int b, int a, int lane, int cut);

template <bool EMIT>
__global__ void __launch_bounds__(256) nms_overflow_pass_kernel(const NmsParams p) {
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int cut = 0;
  if (EMIT) {
    cut = p.ws.cutoff[b];
    if (cut < 0) return;
  } else if (p.ws.cand_count[b] <= p.ws.cap) {
    return;
  }
  // one warp per anchor row, 64 rows per warp: the grid stays small, so the launch costs next to nothing for the
  // images that did not overflow (every block of such an image returns above)
  for (int a = (blockIdx.x * 8 + warp) * kOverflowRows, a_end = min(p.A, a + kOverflowRows); a < a_end; ++a)
    overflow_row<EMIT>(p, b, a, lane, cut);
}

template <bool EMIT>
__device__ __forceinline__ void overflow_row(const NmsParams& p, int b, int a, int lane, int cut) {
  const float* row = p.rows + ((int64_t)b * p.A + a) * p.row_pitch;
  const float obj = p.has_obj ? __ldg(row + 4) : 1.f;
  float raw_max = -INFINITY;
  for (int c = lane; c < p.nc; c += 32) raw_max = fmaxf(raw_max, __ldg(row + p.cls_off + c));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) raw_max = fmaxf(raw_max, __shfl_xor_sync(0xffffffffu, raw_max, o));
  if (!((obj > p.conf) && (raw_max > p.conf))) return;                    // nms.py:48
  uint64_t* keys = p.ws.keys + (int64_t)b * p.ws.cap2;
  uint32_t* hist = p.ws.hist + (int64_t)b * kHistBins;
  for (int c0 = 0; c0 < p.nc; c0 += 32) {
    const int c = c0 + lane;
    const bool cls_ok = (c < p.nc) && ((p.class_mask == nullptr) || (p.class_mask[c] != 0));
    const float sv = (c < p.nc) ? __fmul_rn(__ldg(row + p.cls_off + c), obj) : 0.f;
    const bool hit = cls_ok && (sv > p.conf);
    if (!EMIT) {
      if (hit) atomicAdd(&hist[score_bin(sv)], 1u);
    } else {
      const bool take = hit && (score_bin(sv) >= cut);
      const unsigned m = __ballot_sync(0xffffffffu, take);
      if (m == 0u) continue;
      int slot0 = 0;
      if (lane == 0) slot0 = atomicAdd(&p.ws.cand_count[b], __popc(m));
      slot0 = __shfl_sync(0xffffffffu, slot0, 0);
      if (take) {
        const int my = slot0 + __popc(m & ((1u << lane) - 1u));
        if (my < p.ws.cap) keys[my] = make_key(sv, a * p.nc + c);
      }
    }
  }
}

__global__ void __launch_bounds__(1024) nms_cutoff_kernel(const NmsParams p) {
  __shared__ uint32_t part[1024];
  __shared__ int s_cut;
  const int b = blockIdx.x;
  if (p.ws.cand_count[b] <= p.ws.cap) {
    if (threadIdx.x == 0) p.ws.cutoff[b] = -1;
    return;
  }
  constexpr int PER = kHistBins / 1024;
  const uint32_t* hist = p.ws.hist + (int64_t)b * kHistBins;
  uint32_t mine[PER], tot = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) { mine[j] = hist[threadIdx.x * PER + j]; tot += mine[j]; }
  part[threadIdx.x] = tot;
  if (threadIdx.x == 0) s_cut = 0;
  __syncthreads();
  // suffix sums over threads (Hillis-Steele on 1024 entries)
  for (int o = 1; o < 1024; o <<= 1) {
    const uint32_t add = (threadIdx.x + o < 1024) ? part[threadIdx.x + o] : 0u;
    __syncthreads();
    part[threadIdx.x] += add;
    __syncthreads();
  }
  const uint32_t above = (threadIdx.x + 1 < 1024) ? part[threadIdx.x + 1] : 0u;   // candidates in higher bins than mine
  if (above < (uint32_t)kMaxNms && part[threadIdx.x] >= (uint32_t)kMaxNms) {        // the crossing lies in my bins
    uint32_t acc = above;
    int cut = threadIdx.x * PER;
    for (int j = PER - 1; j >= 0; --j) {
      acc += mine[j];
      if (acc >= (uint32_t)kMaxNms) { cut = threadIdx.x * PER + j; break; }
    }
    s_cut = cut;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    p.ws.cutoff[b] = s_cut;
    p.ws.cand_count[b] = 0;            // the kept bins are re-emitted from scratch
  }
}

// Bitonic network over P (power of two) keys by one block.  Compare-exchange distances below CH stay inside one warp's
// chunk of CH keys, so those passes need only __syncwarp; block barriers are paid for the few long-distance passes alone.
__device__ __forceinline__ void block_bitonic_sort(uint64_t* k, int P) {
  const int CH = min(P, 256);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int size = 2; size <= P; size <<= 1) {
    int j = size >> 1;
    for (; j >= CH; j >>= 1) {
      for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const int i = ((t / j) * 2 * j) + (t % j);
        const int l = i + j;
        const uint64_t x = k[i], y = k[l];
        const bool up = ((i & size) == 0);
        if ((x > y) == up) { k[i] = y; k[l] = x; }
      }
      __syncthreads();
    }
    for (; j > 0; j >>= 1) {
      for (int chunk = warp; chunk * CH < P; chunk += nwarps) {
        const int base = chunk * CH;
        for (int t = lane; t < (CH >> 1); t += 32) {
          const int i = base + ((t / j) * 2 * j) + (t % j);
          const int l = i + j;
          const uint64_t x = k[i], y = k[l];
          const bool up = ((i & size) == 0);
          if ((x > y) == up) { k[i] = y; k[l] = x; }
        }
      }
      __syncwarp();
    }
    __syncthreads();
  }
}

// Full sort of an image's keys (in place).  FALLBACK = second launch of the top-K scheme: only images whose prefix ran out.
template <bool FALLBACK>
__global__ void __launch_bounds__(1024) nms_sort_kernel(const NmsParams p) {
  extern __shared__ uint64_t skeys[];
  const int b = blockIdx.x;
  if (FALLBACK && !p.ws.need_full[b]) return;
  const int taken = p.ws.cand_count[b];
  if (!FALLBACK && taken > p.ws.cap && threadIdx.x == 0) atomicExch(p.ws.overflow, 1);
  const int n = min(taken, p.ws.cap);
  if (n <= 1) return;
  int P = 2;
  while (P < n) P <<= 1;
  uint64_t* g = p.ws.keys + (int64_t)b * p.ws.cap2;
  const bool in_smem = (P <= kSortSmemMax);
  uint64_t* k = in_smem ? skeys : g;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const uint64_t v = (i < n) ? g[i] : ~0ull;  // pad sorts last
    k[i] = v;
  }
  __syncthreads();
  block_bitonic_sort(k, P);
  if (in_smem)
    for (int i = threadIdx.x; i < n; i += blockDim.x) g[i] = k[i];
}

// Top-K prefix: sorts all keys when there are at most kTopK of them (top_n = -1: `keys` is the sorted list); otherwise picks the
// lowest score bin such that the bins from it upwards hold >= kTopK keys, gathers exactly those keys and sorts them into
// `top_keys`.  Every key outside the prefix has a strictly lower score bin, so the prefix is a true prefix of the full order.
__global__ void __launch_bounds__(1024) nms_topk_sort_kernel(const NmsParams p) {
  extern __shared__ uint64_t skeys[];
  __shared__ uint32_t part[1024];
  __shared__ int s_cut, s_m, s_fill;
  const int b = blockIdx.x;
  const int taken = p.ws.cand_count[b];
  if (taken > p.ws.cap && threadIdx.x == 0) atomicExch(p.ws.overflow, 1);
  const int n = min(taken, p.ws.cap);
  uint64_t* g = p.ws.keys + (int64_t)b * p.ws.cap2;
  if (n <= kTopK) {                     // small image: one full sort, as before
    if (threadIdx.x == 0) p.ws.top_n[b] = -1;
    if (n <= 1) return;
    int P = 2;
    while (P < n) P <<= 1;
    for (int i = threadIdx.x; i < P; i += blockDim.x) skeys[i] = (i < n) ? g[i] : ~0ull;
    __syncthreads();
    block_bitonic_sort(skeys, P);
    for (int i = threadIdx.x; i < n; i += blockDim.x) g[i] = skeys[i];
    return;
  }
  constexpr int PER = kHistBins / 1024;
  const uint32_t* hist = p.ws.top_hist + (int64_t)b * kHistBins;
  uint32_t mine[PER], tot = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) { mine[j] = hist[threadIdx.x * PER + j]; tot += mine[j]; }
  part[threadIdx.x] = tot;
  if (threadIdx.x == 0) { s_cut = 0; s_m = 0; s_fill = 0; }
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const uint32_t add = (threadIdx.x + o < 1024) ? part[threadIdx.x + o] : 0u;
    __syncthreads();
    part[threadIdx.x] += add;
    __syncthreads();
  }
  const uint32_t above = (threadIdx.x + 1 < 1024) ? part[threadIdx.x + 1] : 0u;
  if (above < (uint32_t)kTopK && part[threadIdx.x] >= (uint32_t)kTopK) {
    uint32_t acc = above;
    int cut = threadIdx.x * PER;
    for (int j = PER - 1; j >= 0; --j) {
      acc += mine[j];
      if (acc >= (uint32_t)kTopK) { cut = threadIdx.x * PER + j; break; }
    }
    s_cut = cut;
    s_m = (int)acc;
  }
  __syncthreads();
  const int cut = s_cut, m = s_m;
  // the histogram counts every candidate, the key list may have been truncated to `cap` (then the overflow pass re-emitted the
  // best >= 30000): m keys are expected above the cut; if they do not fit the prefix buffer, or the lists disagree, sort everything
  if (m <= 0 || m > kTopCap || taken > p.ws.cap) {
    if (threadIdx.x == 0) { p.ws.top_n[b] = 0; p.ws.need_full[b] = 1; }
    return;
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t key = g[i];
    const float sc = __uint_as_float(0xffffffffu - (uint32_t)(key >> 32));
    if (score_bin(sc) >= cut) {
      const int at = atomicAdd(&s_fill, 1);
      if (at < kTopCap) skeys[at] = key;
    }
  }
  __syncthreads();
  const int got = min(s_fill, kTopCap);
  int P = 2;
  while (P < got) P <<= 1;
  for (int i = got + threadIdx.x; i < P; i += blockDim.x) skeys[i] = ~0ull;
  __syncthreads();
  block_bitonic_sort(skeys, P);
  uint64_t* out = p.ws.top_keys + (int64_t)b * kTopCap;
  for (int i = threadIdx.x; i < got; i += blockDim.x) out[i] = skeys[i];
  if (threadIdx.x == 0) p.ws.top_n[b] = got;
}

constexpr int kGreedyThreads = 512;

// MODE 0: sorted `keys` (full list).  MODE 1: top-K scheme, first pass -- the sorted prefix (or the full list when top_n = -1);
// raises need_full when the prefix is exhausted before max_det boxes are kept.  MODE 2: second pass over the full list, only
// for the images that raised it.
template <int MODE>
__global__ void __launch_bounds__(kGreedyThreads) nms_greedy_kernel(const NmsParams p) {
  extern __shared__ float4 gsm[];
  float4* kept_box = gsm;                                              // [max_det] offset boxes
  float* kept_area = reinterpret_cast<float*>(kept_box + p.max_det);   // [max_det]
  __shared__ float4 ch_box[64];
  __shared__ float ch_area[64];
  __shared__ float4 ch_raw[64];         // un-offset xyxy box (the output)
  __shared__ int ch_cls[64], ch_anchor[64];
  __shared__ float ch_score[64];
  __shared__ int ch_alive[64];
  __shared__ unsigned int ch_mask[64][2];
  __shared__ int ch_out[64];            // output row of each chunk member, -1 when suppressed
  __shared__ int s_kept;
  const int b = blockIdx.x;
  const int n_all = min(min(p.ws.cand_count[b], p.ws.cap), kMaxNms);
  int n = n_all;
  const uint64_t* keys = p.ws.keys + (int64_t)b * p.ws.cap2;
  if (MODE == 1) {
    const int tn = p.ws.top_n[b];
    if (tn >= 0) {
      if (p.ws.need_full[b]) return;         // the prefix could not be built: the second pass does this image
      n = min(tn, n_all);
      keys = p.ws.top_keys + (int64_t)b * kTopCap;
    }
  } else if (MODE == 2) {
    if (!p.ws.need_full[b]) return;
  }
  const int div = p.multi_label ? p.nc : 1;                            // key order = anchor * div + class
  const double thr = p.iou;
  if (threadIdx.x == 0) s_kept = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += 64) {
    const int m = min(64, n - c0);
    const int kept = s_kept;
    if (kept >= p.max_det) break;
    if (threadIdx.x < 64) {
      const int c = threadIdx.x;
      ch_alive[c] = (c < m);
      ch_mask[c][0] = ch_mask[c][1] = 0u;
      if (c < m) {
        const uint64_t key = keys[c0 + c];
        const int order = (int)(key & 0xffffffffu);
        const int anchor = order / div;
        int cls;
        if (p.multi_label) {
          cls = order - anchor * div;
        } else {                                                         // best class: recompute from the row (exact)
          const float* row = p.rows + ((int64_t)b * p.A + anchor) * p.row_pitch;
          const float obj = p.has_obj ? __ldg(row + 4) : 1.f;
          float best = -INFINITY;
          cls = 0;
          for (int cc = 0; cc < p.nc; ++cc) {
            const float sv = __fmul_rn(__ldg(row + p.cls_off + cc), obj);
            if (sv > best) { best = sv; cls = cc; }
          }
        }
        const float4 raw = candidate_box(p, b, anchor);
        float4 bx = raw;
        if (!p.agnostic) {
          const float off = __fmul_rn((float)cls, 4096.f);                // nms.py:94
          bx = make_float4(__fadd_rn(bx.x, off), __fadd_rn(bx.y, off), __fadd_rn(bx.z, off), __fadd_rn(bx.w, off));
        }
        ch_raw[c] = raw;
        ch_cls[c] = cls;
        ch_anchor[c] = anchor;
        ch_score[c] = __uint_as_float(0xffffffffu - (uint32_t)(key >> 32));
        ch_box[c] = bx;
        ch_area[c] = __fmul_rn(__fsub_rn(bx.z, bx.x), __fsub_rn(bx.w, bx.y));
      }
    }
    __syncthreads();
    // (a) candidates of this chunk vs. boxes kept from earlier chunks
    {
      const int c = threadIdx.x & 63;
      if (c < m) {
        const float4 cb = ch_box[c];
        const float ca = ch_area[c];
        for (int k = threadIdx.x >> 6; k < kept; k += kGreedyThreads / 64) {
          const float4 kb = kept_box[k];
          const float w = fmaxf(0.f, __fsub_rn(fminf(kb.z, cb.z), fmaxf(kb.x, cb.x)));
          const float h = fmaxf(0.f, __fsub_rn(fminf(kb.w, cb.w), fmaxf(kb.y, cb.y)));
          const float inter = __fmul_rn(w, h);
          const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(kept_area[k], ca), inter));
          if ((double)ovr > thr) { ch_alive[c] = 0; break; }
        }
      }
    }
    // (b) pairwise suppression inside the chunk: bit j of mask[i] = (i < j and IoU(i,j) > thr)
    for (int pr = threadIdx.x; pr < 64 * 64; pr += kGreedyThreads) {
      const int i = pr >> 6, j = pr & 63;
      if (i < j && j < m) {
        const float4 a = ch_box[i], c = ch_box[j];
        const float w = fmaxf(0.f, __fsub_rn(fminf(a.z, c.z), fmaxf(a.x, c.x)));
        const float h = fmaxf(0.f, __fsub_rn(fminf(a.w, c.w), fmaxf(a.y, c.y)));
        const float inter = __fmul_rn(w, h);
        const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ch_area[i], ch_area[j]), inter));
        if ((double)ovr > thr) atomicOr(&ch_mask[i][j >> 5], 1u << (j & 31));
      }
    }
    __syncthreads();
    // (c) sequential resolve of the chunk (bit masks only), then the survivors are appended in parallel
    if (threadIdx.x == 0) {
      unsigned int rem0 = 0u, rem1 = 0u;
      int k = kept;
      for (int c = 0; c < 64; ++c) {
        const bool removed = (c < 32) ? ((rem0 >> c) & 1u) : ((rem1 >> (c - 32)) & 1u);
        int o = -1;
        if (c < m && k < p.max_det && ch_alive[c] && !removed) {
          rem0 |= ch_mask[c][0];
          rem1 |= ch_mask[c][1];
          o = k++;
        }
        ch_out[c] = o;
      }
      s_kept = k;
    }
    __syncthreads();
    if (threadIdx.x < 64) {
      const int c = threadIdx.x, k = ch_out[c];
      if (k >= 0) {
        kept_box[k] = ch_box[c];
        kept_area[k] = ch_area[c];
        const float4 bx = ch_raw[c];
        float* o = p.out + ((int64_t)b * p.max_det + k) * 6;
        o[0] = bx.x; o[1] = bx.y; o[2] = bx.z; o[3] = bx.w;
        o[4] = ch_score[c];
        o[5] = (float)ch_cls[c];
        p.out_src[((int64_t)b * p.max_det + k) * 2] = ch_anchor[c];
        p.out_src[((int64_t)b * p.max_det + k) * 2 + 1] = ch_cls[c];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.out_count[b] = s_kept;
    if (MODE == 1 && n < n_all && s_kept < p.max_det) p.ws.need_full[b] = 1;   // prefix exhausted: redo on the full list
  }
}

// ------------------------------------------------------------------------------------------------
// Evaluation post-processing of the NMS output, all images at once: Evaler.scale_coords + box_convert + the
// top-left shift of Evaler.convert_to_coco_format (yolov6/core/evaler.py:333-373), in the reference's fp32
// operation order (explicit round-to-nearest ops, so the decimal strings the COCO json gets are identical):
//   x -= pad_x; x /= gain_w; clamp(0, w0)   (same for y with pad_y / gain_h / h0)
//   xc = (x1 + x2) / 2; w = x2 - x1; x_tl = xc - w / 2
// meta [B][6] = (gain_h, gain_w, pad_x, pad_y, h0, w0) per image (shapes[i] of the reference's dataloader).
__global__ void eval_boxes_kernel(const float* __restrict__ det, const int32_t* __restrict__ count, const float* __restrict__ meta,
                                  int B, int max_det, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * max_det) return;
  const int b = i / max_det, j = i - b * max_det;
  float* o = out + (int64_t)i * 6;
  if (j >= count[b]) {
    o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0.f;
    return;
  }
  const float* r = det + (int64_t)i * 6;
  const float4 s = scale_coords_rn(r[0], r[1], r[2], r[3], meta + b * 6);
  const float x1 = s.x, y1 = s.y, x2 = s.z, y2 = s.w;
  const float xc = __fdiv_rn(__fadd_rn(x1, x2), 2.f), yc = __fdiv_rn(__fadd_rn(y1, y2), 2.f);
  const float w = __fsub_rn(x2, x1), hh = __fsub_rn(y2, y1);
  o[0] = __fsub_rn(xc, __fdiv_rn(w, 2.f));
  o[1] = __fsub_rn(yc, __fdiv_rn(hh, 2.f));
  o[2] = w;
  o[3] = hh;
  o[4] = r[4];
  o[5] = r[5];
}

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

static void nms_layout(int32_t B, int32_t A, int32_t nc, int32_t multi_label, NmsWs* ws, int64_t* total, char* base) {
  int64_t cap = multi_label ? (int64_t)A * nc : A;
  if (cap > kMultiCap && multi_label) cap = kMultiCap;
  int64_t cap2 = 2;
  while (cap2 < cap) cap2 <<= 1;
  const int T = (A + kNmsTile - 1) / kNmsTile;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { int64_t o = off; off += align256(bytes); return base ? base + o : (char*)nullptr; };
  ws->cand_count = (int32_t*)take((int64_t)B * 4);
  ws->overflow = (int32_t*)take(4);
  ws->keys = (uint64_t*)take((int64_t)B * cap2 * 8);
  const bool can_overflow = multi_label && (int64_t)A * nc > cap;
  ws->hist = can_overflow ? (uint32_t*)take((int64_t)B * kHistBins * 4) : nullptr;
  ws->cutoff = can_overflow ? (int32_t*)take((int64_t)B * 4) : nullptr;
  ws->top_hist = (uint32_t*)take((int64_t)B * kHistBins * 4);       // adjacent to top_n / need_full: one memset clears all three
  ws->top_n = (int32_t*)take((int64_t)B * 4);
  ws->need_full = (int32_t*)take((int64_t)B * 4);
  ws->top_keys = (uint64_t*)take((int64_t)B * kTopCap * 8);
  ws->cap = (int32_t)cap;
  ws->cap2 = (int32_t)cap2;
  ws->T = T;
  *total = off;
}

}  // namespace yv6

using namespace yv6;

extern "C" int64_t yv6_nms_workspace_bytes(int32_t B, int32_t A, int32_t nc, int32_t multi_label) {
  NmsWs ws;
  int64_t total = 0;
  nms_layout(B, A, nc, multi_label, &ws, &total, nullptr);
  return total;
}

static int nms_launch(yv6_handle* h, NmsParams& p, int32_t B, int32_t A, int32_t nc, float conf_thres, double iou_thres,
                      int32_t agnostic, int32_t multi_label, const uint8_t* class_mask, int32_t max_det, float* out,
                      int32_t* out_count, int32_t* out_src, int32_t* overflow, void* workspace, int64_t workspace_bytes, void* stream) {
  YV6_REQUIRE(out && out_count && out_src && workspace, "nms: null argument");
  YV6_REQUIRE(B > 0 && A > 0 && nc > 0, "nms: bad shape B=%d A=%d nc=%d", B, A, nc);
  YV6_REQUIRE(conf_thres >= 0.f && conf_thres <= 1.f, "nms: conf_thres must be in [0,1]");       // nms.py:50
  YV6_REQUIRE(iou_thres >= 0.0 && iou_thres <= 1.0, "nms: iou_thres must be in [0,1]");          // nms.py:51
  YV6_REQUIRE(max_det > 0 && max_det <= 4096, "nms: max_det=%d out of range (1..4096)", max_det);
  int64_t need = 0;
  const int ml = (multi_label && nc > 1) ? 1 : 0;                                                // nms.py:57
  nms_layout(B, A, nc, ml, &p.ws, &need, reinterpret_cast<char*>(workspace));
  YV6_REQUIRE(workspace_bytes >= need, "nms: workspace too small (%lld < %lld)", (long long)workspace_bytes, (long long)need);
  p.B = B;
  p.A = A;
  p.nc = nc;
  p.no = nc + 5;
  p.conf = conf_thres;
  p.iou = iou_thres;
  p.agnostic = agnostic;
  p.multi_label = ml;
  p.max_det = max_det;
  p.class_mask = class_mask;
  p.out = out;
  p.out_count = out_count;
  p.out_src = out_src;
  if (overflow != nullptr) p.ws.overflow = overflow;
  cudaStream_t s = (cudaStream_t)stream;
  YV6_CHECK_CUDA(cudaMemsetAsync(p.ws.overflow, 0, 4, s));
  YV6_CHECK_CUDA(cudaMemsetAsync(p.ws.cand_count, 0, sizeof(int32_t) * B, s));
  // the row tile of the lane-per-row kernel must fit the CTA's opt-in shared memory (nc <= 220 with 227 KB; wider heads take the generic kernel)
  const size_t sel_smem_bytes = sizeof(float) * 8 * kSelRows * (size_t)(nc | 1);
  const bool rows_mode = !p.has_obj && p.row_pitch == nc && nc % 4 == 0 && sel_smem_bytes <= (size_t)h->max_smem_optin &&
                         (reinterpret_cast<uintptr_t>(p.rows) & 15) == 0;
  if (rows_mode) {
    YV6_CHECK_CUDA(cudaMemsetAsync(p.ws.top_hist, 0, (size_t)(reinterpret_cast<char*>(p.ws.top_keys) - reinterpret_cast<char*>(p.ws.top_hist)), s));
    const size_t smem = sel_smem_bytes;
    dim3 grid((A + 8 * kSelRows - 1) / (8 * kSelRows), B);
    if (!(h->configured & YV6_CFG_SELROWS)) {
      YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_select_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, h->max_smem_optin));
      h->configured |= YV6_CFG_SELROWS;
    }
    nms_select_rows_kernel<<<grid, 256, smem, s>>>(p);
  } else {
    dim3 grid(p.ws.T, B);
    nms_select_kernel<<<grid, kNmsTile, 0, s>>>(p);
  }
  if (p.ws.hist != nullptr) {   // A * nc exceeds the key capacity: keep the max_nms best of an overflowing image (nms.py:90-91)
    YV6_CHECK_CUDA(cudaMemsetAsync(p.ws.hist, 0, sizeof(uint32_t) * (size_t)B * kHistBins, s));
    dim3 g8((A + 8 * kOverflowRows - 1) / (8 * kOverflowRows), B);
    nms_overflow_pass_kernel<false><<<g8, 256, 0, s>>>(p);
    nms_cutoff_kernel<<<B, 1024, 0, s>>>(p);
    nms_overflow_pass_kernel<true><<<g8, 256, 0, s>>>(p);
  }
  if (!(h->configured & YV6_CFG_NMS)) {
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_sort_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSortSmemMax * 8));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_sort_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSortSmemMax * 8));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_topk_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopCap * 8));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_greedy_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 20));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_greedy_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 20));
    YV6_CHECK_CUDA(cudaFuncSetAttribute(nms_greedy_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 20));
    h->configured |= YV6_CFG_NMS;
  }
  const size_t sort_smem = (size_t)std::min<int64_t>(p.ws.cap2, kSortSmemMax) * 8;
  const size_t greedy_smem = (size_t)max_det * 20;
  if (rows_mode) {      // sorted top-K prefix first; the full sort + second greedy pass only touch images whose prefix ran out
    nms_topk_sort_kernel<<<B, 1024, kTopCap * 8, s>>>(p);
    nms_greedy_kernel<1><<<B, kGreedyThreads, greedy_smem, s>>>(p);
    nms_sort_kernel<true><<<B, 1024, sort_smem, s>>>(p);
    nms_greedy_kernel<2><<<B, kGreedyThreads, greedy_smem, s>>>(p);
  } else {
    nms_sort_kernel<false><<<B, 1024, sort_smem, s>>>(p);
    nms_greedy_kernel<0><<<B, kGreedyThreads, greedy_smem, s>>>(p);
  }
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}

extern "C" int yv6_nms_batched(yv6_handle* h, const float* pred, int32_t B, int32_t A, int32_t nc, float conf_thres,
                               double iou_thres, int32_t agnostic, int32_t multi_label, const uint8_t* class_mask,
                               int32_t max_det, float* out, int32_t* out_count, int32_t* out_src, int32_t* overflow,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && pred, "nms: null argument");
  NmsParams p;
  memset(&p, 0, sizeof(p));
  p.rows = pred;
  p.row_pitch = nc + 5;
  p.cls_off = 5;
  p.has_obj = 1;
  return nms_launch(h, p, B, A, nc, conf_thres, iou_thres, agnostic, multi_label, class_mask, max_det, out, out_count, out_src, overflow,
                    workspace, workspace_bytes, stream);
}

extern "C" int yv6_nms_batched_head(yv6_handle* h, const float* cls, const float* reg, int32_t B, int32_t nc, int32_t reg_ch, int32_t nl,
                                    const int32_t* lvl_h, const int32_t* lvl_w, const float* lvl_stride, float conf_thres,
                                    double iou_thres, int32_t agnostic, int32_t multi_label, const uint8_t* class_mask, int32_t max_det,
                                    float* out, int32_t* out_count, int32_t* out_src, int32_t* overflow, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && cls && reg && lvl_h && lvl_w && lvl_stride, "nms_head: null argument");
  YV6_REQUIRE(nl >= 1 && nl <= kNmsMaxLevels && reg_ch >= 4 && reg_ch % 4 == 0, "nms_head: nl=%d reg_ch=%d", nl, reg_ch);
  NmsParams p;
  memset(&p, 0, sizeof(p));
  p.rows = cls;
  p.row_pitch = nc;
  p.cls_off = 0;
  p.has_obj = 0;
  p.reg = reg;
  p.R = reg_ch;
  p.reg_max = reg_ch / 4 - 1;
  p.nl = nl;
  int A = 0;
  for (int l = 0; l < nl; ++l) {
    p.lvl_off[l] = A;
    p.lvl_w[l] = lvl_w[l];
    p.lvl_stride[l] = lvl_stride[l];
    A += lvl_h[l] * lvl_w[l];
  }
  p.lvl_off[nl] = A;
  return nms_launch(h, p, B, A, nc, conf_thres, iou_thres, agnostic, multi_label, class_mask, max_det, out, out_count, out_src, overflow,
                    workspace, workspace_bytes, stream);
}

extern "C" int yv6_eval_boxes(yv6_handle* h, const float* det, const int32_t* count, const float* meta, int32_t B, int32_t max_det,
                              float* out, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && det && count && meta && out && B > 0 && max_det > 0, "eval_boxes: bad argument");
  const int total = B * max_det;
  eval_boxes_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(det, count, meta, B, max_det, out);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
