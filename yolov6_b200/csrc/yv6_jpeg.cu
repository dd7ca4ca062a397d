// yv6_jpeg.cu -- cv2.imread's pixels of baseline / extended sequential Huffman JPEGs (libjpeg-turbo with its defaults),
// a batch of images per call, in three launches:
//   jpeg_entropy_kernel  one CTA per image: unstuff the segment, self-synchronising parallel Huffman decode, DC values,
//                        coefficients in scan order;
//   jpeg_idct_kernel     dequantisation + libjpeg's jpeg_idct_islow into the component sample planes;
//   jpeg_color_kernel    fancy upsampling, YCbCr -> BGR, EXIF orientation, into each image's BGR HWC frame.
//
// Entropy decoding (Weissenberger & Schmidt, ICPP 2018 / HiPC 2021).  The unstuffed scan of T bits is cut into one range
// per thread.  A decoder state at a block boundary is (bit position p, block of the MCU b, restart interval k).  Each
// thread decodes the blocks that start in its range, from the state it is handed, and records the state in which it
// leaves.  Pass 1 hands every thread a guess (its range start, b = 0); every later pass hands thread t the state thread
// t - 1 left in, and a thread decodes again only if that changed.  Two decoders that agree on a state agree from there on,
// and Huffman decoders resynchronise within a few codes, so a few passes settle every boundary; the bound is one pass per
// thread (a sequential decode), and thread 0's state is exact from the start.  A restart marker is an exact sync point:
// whenever p reaches the next interval's start the state becomes (that start, 0, k + 1).  The pad bits before a marker
// may decode as extra blocks; they come after the interval's real blocks and are dropped by count.  A serial scan over the
// threads' block counts and DC sums (reset at each restart) then gives every thread its first block's index in its
// interval and the DC predictors, and a last pass writes the coefficients.
//
// IDCT: jidctint.c's jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) with its post-IDCT range limit, which wraps the
// descaled value modulo 1024 before clamping.  Colour: jdcolor.c's 16-bit fixed-point tables.  Upsampling: jdsample.c's
// h2v1 / h2v2 fancy filters (chroma wider than two samples) and h1v2, replication otherwise; the edges repeat the real
// samples (not the block padding).
#include "yv6_common.cuh"
#include "yv6_handle.h"

namespace yv6 {

constexpr int kJpegThreads = 512;
constexpr int64_t kJpegMinBits = 1024;     // a thread's range is at least this long: ranges longer than the usual
                                           // resynchronisation distance settle in two passes

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// The next 32 bits at bit p of an unstuffed segment (big-endian words, 16 bytes of padding), zeros at and past `end`
// (libjpeg feeds zeros once the data runs out).
__device__ __forceinline__ uint32_t peek32(const uint32_t* __restrict__ w, int64_t p, int64_t end) {
  if (p >= end) return 0;
  const int64_t i = p >> 5;
  const uint64_t v = ((uint64_t)__byte_perm(w[i], 0, 0x0123) << 32) | __byte_perm(w[i + 1], 0, 0x0123);
  uint32_t r = (uint32_t)(v >> (32 - (p & 31)));
  const int64_t valid = end - p;
  if (valid < 32) r &= ~(0xFFFFFFFFu >> valid);
  return r;
}

// One Huffman symbol at p; advances p.  An invalid code sets *err, consumes 16 bits and reads as symbol 0.
__device__ __forceinline__ int huff_sym(const yv6_jpeg_huff& t, const uint32_t* w, int64_t& p, int64_t end, int& err) {
  const uint32_t v = peek32(w, p, end);
  const int e = t.lut[v >> 23];
  if (e) {
    p += e >> 8;
    return e & 255;
  }
  int l = 10;
  while (l <= 16 && (int32_t)(v >> (32 - l)) > t.maxcode[l]) ++l;
  if (l > 16) {
    err = YV6_JPEG_BAD_CODE;
    p += 16;
    return 0;
  }
  p += l;
  return t.vals[((int32_t)(v >> (32 - l)) + t.valoff[l]) & 255];
}

__device__ __forceinline__ int huff_bits(const uint32_t* w, int64_t& p, int64_t end, int s) {
  if (s == 0) return 0;
  const uint32_t v = peek32(w, p, end) >> (32 - s);
  p += s;
  return (int)v < (1 << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v;      // HUFF_EXTEND
}

// One block at p with component tables dc / ac: returns its DC difference; writes its AC coefficients (natural order)
// to blk when blk is not null.  *err: the first defect met.
__device__ __forceinline__ int decode_block(const yv6_jpeg_huff& dc, const yv6_jpeg_huff& ac, const uint32_t* w, int64_t& p,
                                            int64_t end, int16_t* blk, int& err) {
  int s = huff_sym(dc, w, p, end, err);
  if (s > 16) err = YV6_JPEG_BAD_CODE, s = 0;
  const int diff = huff_bits(w, p, end, s);
  for (int k = 1; k < 64;) {
    const int rs = huff_sym(ac, w, p, end, err);
    const int r = rs >> 4;
    s = rs & 15;
    if (s) {
      k += r;
      const int v = huff_bits(w, p, end, s);
      if (k > 63) {
        err = YV6_JPEG_BAD_RUN;
        break;
      }
      if (blk) blk[kZigzag[k]] = (int16_t)v;
      ++k;
    } else if (r == 15) {
      k += 16;
    } else {
      break;
    }
  }
  return diff;
}

struct JpegState {
  int64_t p;
  int b, k;
};

struct JpegTally {               // what a thread's range adds to the intervals it touches
  int jumped;                    // crossed at least one restart
  int n0, n1;                    // blocks before the first restart / after the last
  int dc0[3], dc1[3];            // DC differences summed per component, same split
};

__device__ __forceinline__ void block_comp(const yv6_jpeg_image& im, int b, int& c) {
  const int n0 = im.comp[0].h * im.comp[0].v;
  c = b < n0 ? 0 : b - n0 + 1;
}

// Decodes the blocks that start in [s.p, stop) from state s.  With coef (the write pass): block i of interval k is
// written when it is one of the interval's real blocks (coefficients pre-zeroed), DC predictors starting at dc0, and
// *status gets the first error of a real block.  Returns the tally, leaves s at the exit state.
__device__ JpegTally run_range(const yv6_jpeg_image& im, const yv6_jpeg_huff* tabs, const uint32_t* w, const int64_t* rst,
                               int nint, JpegState& s, int64_t stop, int16_t* coef, int idx, const int* dc0, int* status) {
  JpegTally t{};
  int pred[3] = {dc0 ? dc0[0] : 0, dc0 ? dc0[1] : 0, dc0 ? dc0[2] : 0};
  const int64_t per = (int64_t)im.restart * im.nblk;
  const int64_t nmcu = (int64_t)im.mcux * im.mcuy;
  while (s.p < stop) {
    const int64_t E = rst[s.k + 1];
    int c;
    block_comp(im, s.b, c);
    int err = 0;
    const int64_t real = min((int64_t)im.restart, nmcu - (int64_t)s.k * im.restart) * im.nblk;
    const bool keep = coef && idx < real;
    int16_t* blk = keep ? coef + ((int64_t)s.k * per + idx) * 64 : nullptr;
    const int diff = decode_block(tabs[2 * c], tabs[2 * c + 1], w, s.p, E, blk, err);
    if (keep) {
      pred[c] += diff;
      blk[0] = (int16_t)pred[c];
      if (s.p > E && !err) err = YV6_JPEG_SHORT;
      if (err) atomicCAS(status, 0, err);
    }
    ++idx;
    if (t.jumped) ++t.n1, t.dc1[c] += diff;
    else ++t.n0, t.dc0[c] += diff;
    s.b = s.b + 1 == im.nblk ? 0 : s.b + 1;
    while (s.p >= rst[s.k + 1] && s.k + 1 < nint) {        // restart: an exact state (empty intervals are skipped)
      if (coef && idx < min((int64_t)im.restart, nmcu - (int64_t)s.k * im.restart) * im.nblk) atomicCAS(status, 0, YV6_JPEG_SHORT);
      s.p = rst[s.k + 1], s.k += 1, s.b = 0, idx = 0;
      t.jumped = 1, t.n1 = 0;
      for (int j = 0; j < 3; ++j) t.dc1[j] = 0, pred[j] = 0;
    }
  }
  return t;
}

// Block-wide exclusive scan of one int per thread; returns the prefix, *total the sum.
__device__ __forceinline__ int block_scan(int v, int* warp_sums, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = lane < kJpegThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < kJpegThreads / 32) warp_sums[lane] = s;
  }
  __syncthreads();
  const int before = (wid ? warp_sums[wid - 1] : 0) + x - v;
  total = warp_sums[kJpegThreads / 32 - 1];
  __syncthreads();
  return before;
}

__global__ void __launch_bounds__(kJpegThreads) jpeg_entropy_kernel(const yv6_jpeg_image* __restrict__ imgs,
                                                                   const yv6_jpeg_huff* __restrict__ huff,
                                                                   uint8_t* __restrict__ ws, int32_t* __restrict__ status) {
  __shared__ yv6_jpeg_huff tabs[6];
  __shared__ int warp_sums[kJpegThreads / 32];
  __shared__ int64_t ex_p[kJpegThreads];
  __shared__ int ex_b[kJpegThreads], ex_k[kJpegThreads];
  __shared__ int sc_n[kJpegThreads][2], sc_j[kJpegThreads], sc_dc[kJpegThreads][6];
  const yv6_jpeg_image& im = imgs[blockIdx.x];
  const int tid = threadIdx.x;
  int32_t* st = status + blockIdx.x;
  for (int i = tid; i < im.ncomp * 2 * (int)(sizeof(yv6_jpeg_huff) / 4); i += kJpegThreads) {
    const int tb = i / (int)(sizeof(yv6_jpeg_huff) / 4), o = i % (int)(sizeof(yv6_jpeg_huff) / 4);
    const int src = (tb & 1) ? im.comp[tb >> 1].ac : im.comp[tb >> 1].dc;
    reinterpret_cast<uint32_t*>(&tabs[tb])[o] = reinterpret_cast<const uint32_t*>(&huff[src])[o];
  }
  if (tid == 0) *st = 0;
  const int64_t nmcu = (int64_t)im.mcux * im.mcuy;
  const int nint = (int)((nmcu + im.restart - 1) / im.restart);
  uint8_t* u = ws + im.ws_bytes;
  int64_t* rst = reinterpret_cast<int64_t*>(ws + im.ws_rst);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + im.ws_coef);
  {   // zero the coefficients (the write pass stores only the non-zero ones)
    uint4* z = reinterpret_cast<uint4*>(coef);
    for (int64_t i = tid; i < nmcu * im.nblk * 8; i += kJpegThreads) z[i] = make_uint4(0, 0, 0, 0);
  }

  // ---- unstuff: FF 00 -> FF, fill FFs dropped, RSTn dropped and the next interval's start bit recorded ----
  const uint8_t* d = im.data;
  const int64_t len = im.len;
  int64_t kept = 0, marks = 0;
  for (int64_t base = 0; base < len; base += kJpegThreads * 8) {
    const int64_t i0 = base + (int64_t)tid * 8;
    uint8_t keepv[8];
    int nk = 0, nr = 0;
    int prev = i0 > 0 && i0 - 1 < len ? d[i0 - 1] : 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t i = i0 + j;
      const int x = i < len ? d[i] : -1;
      const int next = i + 1 < len ? d[i + 1] : -1;
      const bool rstm = prev == 0xFF && x >= 0xD0 && x <= 0xD7;
      const bool drop = x < 0 || (x == 0 && prev == 0xFF) || (x == 0xFF && next != 0) || rstm;
      keepv[j] = !drop;
      nk += !drop;
      nr += rstm;
      prev = x;
    }
    int tk, tr;
    const int pk = block_scan(nk, warp_sums, tk);
    const int pr = block_scan(nr, warp_sums, tr);
    int64_t o = kept + pk, r = marks + pr;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t i = i0 + j;
      if (i >= len) break;
      if (keepv[j]) u[o++] = d[i];
      else if (i > 0 && d[i - 1] == 0xFF && d[i] >= 0xD0 && d[i] <= 0xD7 && ++r < nint) rst[r] = o * 8;
    }
    kept += tk, marks += tr;
  }
  if (tid < 16) u[kept + tid] = 0;
  if (tid == 0) rst[0] = 0;
  for (int64_t k = min(marks, (int64_t)nint - 1) + 1 + tid; k <= nint; k += kJpegThreads) rst[k] = kept * 8;
  __syncthreads();

  // ---- self-synchronising decode ----
  const uint32_t* w = reinterpret_cast<const uint32_t*>(u);
  const int64_t T = kept * 8;
  const int64_t sub = max(kJpegMinBits, (T + kJpegThreads - 1) / kJpegThreads);
  const int act = (int)max((int64_t)1, (T + sub - 1) / sub);        // threads with a range; the rest stay idle
  const int64_t lo = min((int64_t)tid * sub, T), hi = min(lo + sub, T);
  JpegState in;
  {
    int a = 0, b = nint;                        // the interval holding lo: last k with rst[k] <= lo
    while (b - a > 1) {
      const int m = (a + b) >> 1;
      if (rst[m] <= lo) a = m;
      else b = m;
    }
    in = JpegState{lo, 0, a};
  }
  if (tid == 0) in = JpegState{0, 0, 0};
  bool todo = true;
  JpegTally tally{};
  JpegState out = in;
  for (int pass = 0; pass < kJpegThreads; ++pass) {
    if (todo) {
      out = in;
      tally = run_range(im, tabs, w, rst, nint, out, hi, nullptr, 0, nullptr, st);
      todo = false;
    }
    ex_p[tid] = out.p, ex_b[tid] = out.b, ex_k[tid] = out.k;
    __syncthreads();
    if (tid > 0 && tid < act && (ex_p[tid - 1] != in.p || ex_b[tid - 1] != in.b || ex_k[tid - 1] != in.k)) {
      in = JpegState{ex_p[tid - 1], ex_b[tid - 1], ex_k[tid - 1]};
      todo = true;
    }
    if (!__syncthreads_or(todo)) break;
  }

  // ---- each thread's first block index in its interval and DC predictors: serial scan over the threads ----
  sc_j[tid] = tally.jumped, sc_n[tid][0] = tally.n0, sc_n[tid][1] = tally.n1;
  for (int j = 0; j < 3; ++j) sc_dc[tid][j] = tally.dc0[j], sc_dc[tid][3 + j] = tally.dc1[j];
  __syncthreads();
  if (tid == 0) {
    int n = 0, dc[3] = {0, 0, 0};
    for (int t = 0; t < act; ++t) {
      const int j = sc_j[t], n0 = sc_n[t][0], n1 = sc_n[t][1];
      int e[6];
      for (int c = 0; c < 6; ++c) e[c] = sc_dc[t][c];
      sc_n[t][0] = n;
      for (int c = 0; c < 3; ++c) sc_dc[t][c] = dc[c];
      if (j) {
        n = n1;
        for (int c = 0; c < 3; ++c) dc[c] = e[3 + c];
      } else {
        n += n0;
        for (int c = 0; c < 3; ++c) dc[c] += e[c];
      }
    }
    const int klast = ex_k[act - 1];      // the end of the stream: every interval reached, the last one complete
    if (klast < nint - 1 || n < min((int64_t)im.restart, nmcu - (int64_t)klast * im.restart) * im.nblk) atomicCAS(st, 0, YV6_JPEG_SHORT);
  }
  __syncthreads();

  // ---- write pass ----
  JpegState s = in;
  if (tid < act) run_range(im, tabs, w, rst, nint, s, hi, coef, sc_n[tid][0], sc_dc[tid], st);
}

// libjpeg's jidctint.c 1-D pass on 8 values; `shift` is the descale.
__device__ __forceinline__ void idct8(int (&x)[8], int shift) {
  const int z1a = (x[2] + x[6]) * 4433;
  const int tmp2 = z1a - x[6] * 15137, tmp3 = z1a + x[2] * 6270;
  const int tmp0 = (x[0] + x[4]) * 8192, tmp1 = (x[0] - x[4]) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  int z1 = o0 + o3, z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const int z5 = (z3 + z4) * 9633;
  o0 *= 2446, o1 *= 16819, o2 *= 25172, o3 *= 12299;
  z1 *= -7373, z2 *= -20995, z3 = z3 * -16069 + z5, z4 = z4 * -3196 + z5;
  o0 += z1 + z3, o1 += z2 + z4, o2 += z2 + z3, o3 += z1 + z4;
  const int r = 1 << (shift - 1);
  x[0] = (t10 + o3 + r) >> shift, x[7] = (t10 - o3 + r) >> shift;
  x[1] = (t11 + o2 + r) >> shift, x[6] = (t11 - o2 + r) >> shift;
  x[2] = (t12 + o1 + r) >> shift, x[5] = (t12 - o1 + r) >> shift;
  x[3] = (t13 + o0 + r) >> shift, x[4] = (t13 - o0 + r) >> shift;
}

__device__ __forceinline__ uint8_t range_limit(int v) {     // idct range_limit[v & RANGE_MASK] (centre 128)
  const int j = v & 1023;
  return (uint8_t)(j < 128 ? j + 128 : j < 512 ? 255 : j < 896 ? 0 : j - 896);
}

// thread = one 8x8 block of image blockIdx.y.
__global__ void __launch_bounds__(256) jpeg_idct_kernel(const yv6_jpeg_image* __restrict__ imgs, uint8_t* __restrict__ ws) {
  const yv6_jpeg_image& im = imgs[blockIdx.y];
  __shared__ int q[3][64];
  for (int i = threadIdx.x; i < im.ncomp * 64; i += blockDim.x) q[i / 64][i % 64] = im.comp[i / 64].q[i % 64];
  __syncthreads();
  const int64_t nblocks = (int64_t)im.mcux * im.mcuy * im.nblk;
  const int16_t* coef = reinterpret_cast<const int16_t*>(ws + im.ws_coef);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < nblocks; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = g / im.nblk;
    const int b = (int)(g - m * im.nblk);
    int c;
    block_comp(im, b, c);
    const yv6_jpeg_comp& cp = im.comp[c];
    const int bb = c ? 0 : b;
    const int my = (int)(m / im.mcux), mx = (int)(m - (int64_t)my * im.mcux);
    const int by = my * cp.v + bb / cp.h, bx = mx * cp.h + bb % cp.h;
    int x[8][8];
    const uint4* src = reinterpret_cast<const uint4*>(coef + g * 64);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const uint4 v = src[r];
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        x[r][2 * j] = (int)(int16_t)(u[j] & 0xFFFF) * q[c][r * 8 + 2 * j];
        x[r][2 * j + 1] = (int)(int16_t)(u[j] >> 16) * q[c][r * 8 + 2 * j + 1];
      }
    }
#pragma unroll
    for (int col = 0; col < 8; ++col) {         // pass 1: columns, descale by CONST_BITS - PASS1_BITS
      int v[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) v[r] = x[r][col];
      idct8(v, 11);
#pragma unroll
      for (int r = 0; r < 8; ++r) x[r][col] = v[r];
    }
    uint8_t* dst = ws + cp.plane + ((int64_t)by * 8) * (cp.bw * 8) + bx * 8;
#pragma unroll
    for (int r = 0; r < 8; ++r) {               // pass 2: rows, descale by CONST_BITS + PASS1_BITS + 3
      idct8(x[r], 18);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) lo |= (uint32_t)range_limit(x[r][j]) << (8 * j), hi |= (uint32_t)range_limit(x[r][4 + j]) << (8 * j);
      *reinterpret_cast<uint2*>(dst + (int64_t)r * cp.bw * 8) = make_uint2(lo, hi);
    }
  }
}

// libjpeg-turbo's upsampled chroma sample at luma pixel (y, x) (jdsample.c, do_fancy_upsampling on).
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ ws, const yv6_jpeg_comp& cp, int hf, int vf, int y, int x) {
  const uint8_t* P = ws + cp.plane;
  const int pitch = cp.bw * 8;
  auto at = [&](int r, int c) { return (int)__ldg(P + (int64_t)r * pitch + c); };
  if (hf == 1 && vf == 1) return at(y, x);
  if (hf == 2 && vf == 1 && cp.dw > 2) {
    const int cx = x >> 1, odd = x & 1;
    const int nx = odd ? min(cx + 1, cp.dw - 1) : max(cx - 1, 0);
    return (3 * at(y, cx) + at(y, nx) + 1 + odd) >> 2;
  }
  if (hf == 1 && vf == 2) {
    const int cy = y >> 1, odd = y & 1;
    const int ny = odd ? min(cy + 1, cp.dh - 1) : max(cy - 1, 0);
    return (3 * at(cy, x) + at(ny, x) + 1 + odd) >> 2;
  }
  if (hf == 2 && vf == 2 && cp.dw > 2) {
    const int cy = y >> 1, cx = x >> 1, oy = y & 1, ox = x & 1;
    const int ny = oy ? min(cy + 1, cp.dh - 1) : max(cy - 1, 0);
    const int nx = ox ? min(cx + 1, cp.dw - 1) : max(cx - 1, 0);
    const int s0 = 3 * at(cy, cx) + at(ny, cx), s1 = 3 * at(cy, nx) + at(ny, nx);
    return (3 * s0 + s1 + 8 - ox) >> 4;
  }
  return at(y / vf, x / hf);
}

// thread = one output pixel of image blockIdx.y (after orientation).
__global__ void __launch_bounds__(256) jpeg_color_kernel(const yv6_jpeg_image* __restrict__ imgs, const uint8_t* __restrict__ ws) {
  const yv6_jpeg_image& im = imgs[blockIdx.y];
  const int H = im.height, W = im.width, o = im.orientation;
  const int oh = o >= 5 ? W : H, ow = o >= 5 ? H : W;
  const int hm = max(im.comp[0].h, max(im.comp[1].h, im.comp[2].h)), vm = max(im.comp[0].v, max(im.comp[1].v, im.comp[2].v));
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)oh * ow; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i - (int64_t)oy * ow);
    int y, x;
    switch (o) {
      case 2: y = oy, x = W - 1 - ox; break;
      case 3: y = H - 1 - oy, x = W - 1 - ox; break;
      case 4: y = H - 1 - oy, x = ox; break;
      case 5: y = ox, x = oy; break;
      case 6: y = H - 1 - ox, x = oy; break;
      case 7: y = H - 1 - ox, x = W - 1 - oy; break;
      case 8: y = ox, x = W - 1 - oy; break;
      default: y = oy, x = ox;
    }
    const int Y = __ldg(ws + im.comp[0].plane + (int64_t)y * (im.comp[0].bw * 8) + x);
    uint8_t* dst = im.out + i * 3;
    if (im.ncomp == 1) {
      dst[0] = dst[1] = dst[2] = (uint8_t)Y;
      continue;
    }
    const int cb = chroma(ws, im.comp[1], hm / im.comp[1].h, vm / im.comp[1].v, y, x) - 128;
    const int cr = chroma(ws, im.comp[2], hm / im.comp[2].h, vm / im.comp[2].v, y, x) - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);              // FIX(1.40200)
    const int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);  // FIX(0.34414), FIX(0.71414)
    const int b = Y + ((116130 * cb + 32768) >> 16);             // FIX(1.77200)
    dst[0] = (uint8_t)min(max(b, 0), 255), dst[1] = (uint8_t)min(max(g, 0), 255), dst[2] = (uint8_t)min(max(r, 0), 255);
  }
}

}  // namespace yv6

using namespace yv6;

static int64_t align16(int64_t v) { return (v + 15) & ~(int64_t)15; }

extern "C" int64_t yv6_jpeg_workspace_bytes(yv6_jpeg_image* imgs, int32_t n) {
  if (!imgs || n < 0) {
    yv6_set_error("jpeg_workspace_bytes: bad argument");
    return -1;
  }
  int64_t coef = 0;
  for (int i = 0; i < n; ++i) {
    yv6_jpeg_image& im = imgs[i];
    if (im.height < 1 || im.width < 1 || (im.ncomp != 1 && im.ncomp != 3) || im.orientation < 1 || im.orientation > 8 ||
        im.restart < 0 || im.len < 0) {
      yv6_set_error("jpeg_workspace_bytes: image %d: bad record", i);
      return -1;
    }
    if (im.ncomp == 1) im.comp[0].h = im.comp[0].v = 1;
    for (int c = im.ncomp; c < 3; ++c) im.comp[c] = im.comp[0];
    int hm = 1, vm = 1;
    im.nblk = 0;
    for (int c = 0; c < im.ncomp; ++c) {
      hm = im.comp[c].h > hm ? im.comp[c].h : hm, vm = im.comp[c].v > vm ? im.comp[c].v : vm;
      im.nblk += im.comp[c].h * im.comp[c].v;
    }
    if (im.nblk > 10 || (im.ncomp == 3 && (im.comp[1].h != 1 || im.comp[1].v != 1 || im.comp[2].h != 1 || im.comp[2].v != 1))) {
      yv6_set_error("jpeg_workspace_bytes: image %d: unsupported sampling", i);
      return -1;
    }
    im.mcux = (im.width + 8 * hm - 1) / (8 * hm), im.mcuy = (im.height + 8 * vm - 1) / (8 * vm);
    const int64_t nmcu = (int64_t)im.mcux * im.mcuy;
    if (im.restart == 0 || im.restart > nmcu) im.restart = (int32_t)nmcu;
    for (int c = 0; c < im.ncomp; ++c) {
      yv6_jpeg_comp& cp = im.comp[c];
      cp.bw = im.mcux * cp.h, cp.bh = im.mcuy * cp.v;
      cp.dw = (int32_t)(((int64_t)im.width * cp.h + hm - 1) / hm), cp.dh = (int32_t)(((int64_t)im.height * cp.v + vm - 1) / vm);
    }
    im.ws_coef = coef;
    coef += nmcu * im.nblk * 128;
  }
  int64_t off = align16(coef);
  for (int i = 0; i < n; ++i) {
    yv6_jpeg_image& im = imgs[i];
    const int64_t nmcu = (int64_t)im.mcux * im.mcuy;
    im.ws_bytes = off, off = align16(off + im.len + 16);
    im.ws_rst = off, off = align16(off + 8 * ((nmcu + im.restart - 1) / im.restart + 1));
    for (int c = 0; c < im.ncomp; ++c) im.comp[c].plane = off, off = align16(off + (int64_t)im.comp[c].bw * im.comp[c].bh * 64);
    for (int c = im.ncomp; c < 3; ++c) im.comp[c].plane = im.comp[0].plane;
  }
  return off;
}

extern "C" int yv6_jpeg_decode(yv6_handle* h, const yv6_jpeg_image* imgs, int32_t n, const yv6_jpeg_huff* huff, void* workspace,
                               int32_t* status, void* stream) {
  yv6_device_guard _dev(h);
  YV6_REQUIRE(h && n >= 0 && (n == 0 || (imgs && huff && workspace && status)), "jpeg_decode: bad argument");
  YV6_REQUIRE(n <= 65535, "jpeg_decode: %d images exceed one launch", n);
  YV6_REQUIRE(((uintptr_t)workspace & 15) == 0, "jpeg_decode: the workspace must be 16-byte aligned");
  if (n == 0) return YV6_OK;
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* ws = (uint8_t*)workspace;
  jpeg_entropy_kernel<<<n, kJpegThreads, 0, s>>>(imgs, huff, ws, status);
  YV6_CHECK_CUDA(cudaGetLastError());
  jpeg_idct_kernel<<<dim3(2 * h->num_sms, n), 256, 0, s>>>(imgs, ws);
  YV6_CHECK_CUDA(cudaGetLastError());
  jpeg_color_kernel<<<dim3(2 * h->num_sms, n), 256, 0, s>>>(imgs, ws);
  YV6_CHECK_CUDA(cudaGetLastError());
  return YV6_OK;
}
