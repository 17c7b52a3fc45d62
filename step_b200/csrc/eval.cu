// eval.cu -- frame-mAP on the device: get_ava_performance.run_evaluation (PascalDetectionEvaluator at IoU 0.5) over the
// rows test.py:210-218 would write to its CSV file, without the file.
//
// step_eval_append rounds each detection as the CSV round trip does ('{:.4}' then float()) and appends the rows to a
// device store in the order they would have been written.  step_eval_run then:
//   1. sorts the rows by (class, score descending, image order descending), stably: the class-level order of
//      ObjectDetectionEvaluation.evaluate, whose argsort is a stable ascending argsort reversed under the tie contract;
//   2. sorts that sequence stably by (class, image): each (image, class) segment then holds its rows by descending
//      score, equal scores in row order;
//   3. matches each segment greedily against the image's ground truth of the class (per_image_evaluation.py:461-474),
//      visiting equal scores from the last row to the first (the reversed stable argsort) and keeping the first 10,000;
//   4. per class, walks the order of step 1: precision and recall, the suffix maximum of the precision, and the AP terms
//      summed in numpy's pairwise order.
// Sorts are LSD radix sorts (8-bit digits, stable).  The file is built with -fmad=false: every float64 operation of
// np_box_ops.iou and metrics.py is rounded on its own.
#include <limits.h>

#include "common.cuh"

namespace step {

constexpr int kScoreZero = 756001;               // code of +-0; positive scores above it, negative ones below
constexpr int kScoreTop = 2 * kScoreZero + 1;    // +inf
constexpr unsigned kScoreMax = (1u << 21) - 1;   // codes fit 21 bits
constexpr int kMaxPerSegment = 10000;            // np_box_list_ops.non_max_suppression's max_output_size
constexpr int kSortThreads = 256;                // one thread per digit value
constexpr int kSortItems = 16;
constexpr int kSortTile = kSortThreads * kSortItems;
constexpr int kApThreads = 1024;
constexpr int kPairwiseLeaf = 128;

// ---- exact '{:.4}' rounding of a float32 ----
// m * 10^q with m in [1000, 9999] is the value rounded to 4 significant digits (ties to even on the exact binary value);
// the result is the double nearest to it, which is what float() of the printed text returns.

__host__ __device__ inline double p10(int k) {  // exact for 0 <= k <= 22
  double r = 1.0;
  for (int i = 0; i < k; ++i) r *= 10.0;
  return r;
}

__host__ __device__ inline unsigned __int128 pow_u128(unsigned b, int k) {
  unsigned __int128 r = 1;
  for (int i = 0; i < k; ++i) r *= b;
  return r;
}

// Round-half-even of the exact value hi + d, where d has the sign s (-1, 0, 1) and is smaller than half an ulp of hi.
__host__ __device__ inline long long rne_hi(double hi, int s) {
  const double fl = floor(hi), f = hi - fl;
  if (f > 0.5) return (long long)fl + 1;
  if (f < 0.5) return (long long)fl;
  if (s > 0) return (long long)fl + 1;
  if (s < 0) return (long long)fl;
  const long long n = (long long)fl;
  return (n & 1) ? n + 1 : n;
}

// x = a * 10^k for a > 0 and |k| <= 22, as its rounded value and the sign of the rounding error.
__host__ __device__ inline void scale_fast(double a, int k, double* hi, int* s) {
  if (k >= 0) {
    const double P = p10(k);
    *hi = a * P;
    const double lo = fma(a, P, -*hi);            // the exact error of the product
    *s = lo > 0 ? 1 : lo < 0 ? -1 : 0;
  } else {
    const double P = p10(-k);
    *hi = a / P;
    const double r = fma(-*hi, P, a);             // exact remainder: x - hi = r / P
    *s = r > 0 ? 1 : r < 0 ? -1 : 0;
  }
}

// The 4-digit mantissa of a > 0 at decimal exponent e (a in [10^e, 10^(e+1)) after the adjustment), as the integer m
// and the decade test: -1 if a * 10^(3-e) < 1000, 1 if >= 10000, 0 otherwise.  Exact for every finite float32.
__host__ __device__ inline int mantissa4(double a, int e, long long* m) {
  const int k = 3 - e;
  if (k >= -22 && k <= 22) {
    double hi; int s;
    scale_fast(a, k, &hi, &s);
    if (hi < 1000.0 || (hi == 1000.0 && s < 0)) return -1;
    if (hi > 10000.0 || (hi == 10000.0 && s >= 0)) return 1;
    *m = rne_hi(hi, s);
    return 0;
  }
  // a = M * 2^E exactly, M < 2^24 for a float32
  int ex;
  const double fr = frexp(a, &ex);
  unsigned long long M = (unsigned long long)ldexp(fr, 53);
  int E = ex - 53;
  while (!(M & 1)) { M >>= 1; ++E; }
  unsigned long long n;
  bool up;
  if (k > 0) {  // x = M * 5^k * 2^(E + k), E + k < 0 here
    const unsigned __int128 N = (unsigned __int128)M * pow_u128(5, k);
    const int sh = -(E + k);
    if (sh <= 0) return 1;
    if (sh >= 127) return -1;
    const unsigned __int128 q = N >> sh, rem = N - (q << sh), half = (unsigned __int128)1 << (sh - 1);
    if (q < 1000) return -1;
    if (q >= 10000) return 1;
    n = (unsigned long long)q;
    up = rem > half || (rem == half && (n & 1));
  } else {      // x = (M * 2^E) / 10^-k, E >= 0 here (a >= 1e26 is an integer)
    const unsigned __int128 V = (unsigned __int128)M << E, D = pow_u128(10, -k);
    const unsigned __int128 q = V / D, rem = V - q * D;
    if (q < 1000) return -1;
    if (q >= 10000) return 1;
    n = (unsigned long long)q;
    up = 2 * rem > D || (2 * rem == D && (n & 1));
  }
  *m = (long long)(n + (up ? 1 : 0));
  return 0;
}

// The double nearest m * 10^q, 1000 <= m <= 9999, -48 <= q <= 35: one correctly rounded operation on exact operands,
// or (q < -22) a long division by 5^-q.
__host__ __device__ inline double decimal_to_double(long long m, int q) {
  const double dm = (double)m;
  if (q >= 0 && q <= 22) return dm * p10(q);
  if (q > 22) return (dm * p10(q - 22)) * 1e22;  // m * 5^(q-22) < 2^53: the first product is exact
  if (q >= -22) return dm / p10(-q);
  const int K = -q;
  const unsigned __int128 D = pow_u128(5, K);
  unsigned __int128 r = (unsigned __int128)m;
  unsigned long long Q = 0;
  int bits = 0;  // m / 5^K = (Q + r / D) * 2^-bits
  while (Q < (1ull << 53)) {
    r <<= 1; Q <<= 1; ++bits;
    if (r >= D) { r -= D; Q |= 1; }
  }
  unsigned long long mant = Q >> 1;
  if ((Q & 1) && (r != 0 || (mant & 1))) ++mant;  // round bit, sticky bit (an exact half cannot occur: D is odd)
  return ldexp((double)mant, -(bits - 1) - K);
}

// '{:.4}'.format(float(f)) parsed by float(), and an integer code whose order is the order of the rounded values
// (equal codes <=> equal values; NaN gets -1, -inf 0, +inf kScoreTop).
__host__ __device__ inline double round4(float f, int* code) {
  const double v = (double)f;
  if (v != v) { *code = -1; return v; }
  if (v == 0.0) { *code = kScoreZero; return v; }
  if (isinf(v)) { *code = v > 0 ? kScoreTop : 0; return v; }
  const double a = fabs(v);
  int ex;
  frexp(a, &ex);
  int e = (int)floor((ex - 1) * 0.30102999566398120);  // floor(log10(a)) or one below
  long long m = 0;
  for (int it = 0; it < 4; ++it) {
    const int d = mantissa4(a, e, &m);
    if (d == 0) break;
    e += d;
  }
  if (m == 10000) { m = 1000; ++e; }
  const int q = e - 3;
  const double r = decimal_to_double(m, q);
  const int c = (q + 48) * 9000 + (int)(m - 1000);
  *code = v > 0 ? kScoreZero + 1 + c : kScoreZero - 1 - c;
  return v > 0 ? r : -r;
}

// ---- block scans ----
template <int NT>
__device__ __forceinline__ int2 block_incl_scan2(int2 v, int2* total) {
  __shared__ int2 warp_tot[NT / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, v.x, o), b = __shfl_up_sync(0xffffffffu, v.y, o);
    if (lane >= o) { v.x += a; v.y += b; }
  }
  if (lane == 31) warp_tot[w] = v;
  __syncthreads();
  if (w == 0) {
    int2 t = lane < NT / 32 ? warp_tot[lane] : make_int2(0, 0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, t.x, o), b = __shfl_up_sync(0xffffffffu, t.y, o);
      if (lane >= o) { t.x += a; t.y += b; }
    }
    if (lane < NT / 32) warp_tot[lane] = t;
  }
  __syncthreads();
  if (w > 0) { v.x += warp_tot[w - 1].x; v.y += warp_tot[w - 1].y; }
  *total = warp_tot[NT / 32 - 1];
  __syncthreads();
  return v;
}

// ---- append ----
__global__ void __launch_bounds__(1024) eval_append_kernel(step_eval_append_params p) {
  __shared__ int s_kept, s_read;
  const int tid = threadIdx.x;
  const step_eval_rows& R = p.rows;
  if (tid == 0) { s_kept = R.counters[0]; s_read = R.counters[1]; }
  __syncthreads();
  for (int b = 0; b < p.B; ++b) {
    const int im = p.img[b];
    if (im < 0) continue;
    const int n = min(max(p.count[b], 0), p.cap);
    for (int k0 = 0; k0 < n; k0 += blockDim.x) {
      const int k = k0 + tid;
      int read = 0, keep = 0, cls = -1, sc = 0;
      double box[4] = {0, 0, 0, 0}, score = 0;
      if (k < n) {
        const float* d = p.det + ((size_t)b * p.cap + k) * 8;
        const float cf = d[5];
        const int c = (int)cf;
        cls = (cf >= 0.0f && c < p.ncls && (float)c == cf) ? p.class_of[c] : -1;
        if (cls >= 0) {
          read = 1;
          int unused;
          const double x1 = round4(d[0], &unused), y1 = round4(d[1], &unused);
          const double x2 = round4(d[2], &unused), y2 = round4(d[3], &unused);
          score = round4(d[4], &sc);
          box[0] = y1; box[1] = x1; box[2] = y2; box[3] = x2;   // the evaluator's [y1, x1, y2, x2]
          keep = (y1 < y2) && (x1 < x2) && score > -10.0;       // _remove_invalid_boxes, filter_scores_greater_than
        }
      }
      int2 tot;
      const int2 inc = block_incl_scan2<1024>(make_int2(read, keep), &tot);
      if (read) atomicMin(&R.img_first[im], s_read + inc.x - 1);
      if (keep) {
        const long long r = (long long)s_kept + inc.y - 1;
        if (r < R.capacity) {
          reinterpret_cast<double4*>(R.box)[r] = make_double4(box[0], box[1], box[2], box[3]);
          R.score[r] = score;
          R.scode[r] = sc;
          R.img[r] = im;
          R.cls[r] = cls;
        }
      }
      __syncthreads();
      if (tid == 0) { s_read += tot.x; s_kept += tot.y; }
      __syncthreads();
    }
  }
  if (tid == 0) { R.counters[0] = s_kept; R.counters[1] = s_read; }
}

// ---- stable LSD radix sort of (64-bit key, 32-bit value) ----
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const unsigned long long* keys, int n, int shift, int* hist) {
  __shared__ int h[256];
  const int tid = threadIdx.x;
  h[tid] = 0;
  __syncthreads();
  const int base = blockIdx.x * kSortTile;
  for (int r = 0; r < kSortItems; ++r) {
    const int i = base + r * kSortThreads + tid;
    if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255], 1);
  }
  __syncthreads();
  hist[tid * gridDim.x + blockIdx.x] = h[tid];
}

// exclusive scan of m counts in place, one CTA
__global__ void __launch_bounds__(1024) exclusive_scan_kernel(int* a, int m) {
  const int tid = threadIdx.x, per = (m + 1023) / 1024, lo = min(tid * per, m), hi = min(lo + per, m);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += a[i];
  int2 tot;
  const int inc = block_incl_scan2<1024>(make_int2(s, 0), &tot).x;
  int run = inc - s;
  for (int i = lo; i < hi; ++i) { const int v = a[i]; a[i] = run; run += v; }
}

__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const unsigned long long* keys, const uint32_t* vals,
                                                                     int n, int shift, const int* offs,
                                                                     unsigned long long* okeys, uint32_t* ovals) {
  __shared__ int base_of[256], run[256];
  __shared__ int wcnt[kSortThreads / 32][256], wpre[kSortThreads / 32][256];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  base_of[tid] = offs[tid * gridDim.x + blockIdx.x];
  run[tid] = 0;
  for (int q = 0; q < kSortThreads / 32; ++q) wcnt[q][tid] = 0;
  __syncthreads();
  const int base = blockIdx.x * kSortTile;
  for (int r = 0; r < kSortItems; ++r) {
    const int i = base + r * kSortThreads + tid;
    const bool valid = i < n;
    unsigned long long k = 0;
    uint32_t v = 0;
    int d = 256;
    if (valid) { k = keys[i]; v = vals[i]; d = (int)((k >> shift) & 255); }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int below = __popc(peers & ((1u << lane) - 1));
    if (valid && below == 0) wcnt[w][d] = __popc(peers);
    __syncthreads();
    {  // thread tid owns digit tid: warps in order, after the earlier rounds
      int s = run[tid];
      for (int q = 0; q < kSortThreads / 32; ++q) { const int c = wcnt[q][tid]; wpre[q][tid] = s; s += c; wcnt[q][tid] = 0; }
      run[tid] = s;
    }
    __syncthreads();
    if (valid) {
      const int pos = base_of[d] + wpre[w][d] + below;
      okeys[pos] = k;
      ovals[pos] = v;
    }
  }
}

// Sorts (k0, v0) by bits [0, bits) of the keys; returns true when the result is in (k1, v1).
static int radix_sort(unsigned long long* k0, uint32_t* v0, unsigned long long* k1, uint32_t* v1, int n, int bits, int* hist,
                      cudaStream_t st, bool* in_second) {
  const int nb = ceil_div(n, kSortTile);
  bool second = false;
  for (int shift = 0; shift < bits; shift += 8) {
    unsigned long long* ki = second ? k1 : k0;
    uint32_t* vi = second ? v1 : v0;
    unsigned long long* ko = second ? k0 : k1;
    uint32_t* vo = second ? v0 : v1;
    radix_hist_kernel<<<nb, kSortThreads, 0, st>>>(ki, n, shift, hist);
    STEP_LAUNCH_CHECK("eval radix_hist_kernel");
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(hist, 256 * nb);
    STEP_LAUNCH_CHECK("eval exclusive_scan_kernel");
    radix_scatter_kernel<<<nb, kSortThreads, 0, st>>>(ki, vi, n, shift, hist, ko, vo);
    STEP_LAUNCH_CHECK("eval radix_scatter_kernel");
    second = !second;
  }
  *in_second = second;
  return 0;
}

// ---- evaluate ----
__global__ void eval_init_kernel(int* cls_start, int* cls_end, int n_classes, unsigned char* taken, int n_gt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_classes) { cls_start[i] = 0; cls_end[i] = 0; }
  if (i < n_gt) taken[i] = 0;
}

// class-level key: class, score descending, image order descending (the row order stays within equal keys)
__global__ void class_key_kernel(step_eval_rows R, int n, unsigned long long* keys, uint32_t* vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long first = (unsigned)R.img_first[R.img[i]];
  keys[i] = ((unsigned long long)R.cls[i] << 52) | ((unsigned long long)(kScoreMax - (unsigned)R.scode[i]) << 31) |
            (0x7fffffffull - first);
  vals[i] = (uint32_t)i;
}

__global__ void segment_key_kernel(step_eval_rows R, int n, const uint32_t* order, unsigned long long* keys, uint32_t* vals) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t r = order[j];
  keys[j] = ((unsigned long long)R.cls[r] << 20) | (unsigned long long)R.img[r];
  vals[j] = r;
}

__device__ __forceinline__ double np_max(double a, double b) { return (a >= b || a != a) ? a : b; }  // np.maximum
__device__ __forceinline__ double np_min(double a, double b) { return (a <= b || a != a) ? a : b; }  // np.minimum

// np_box_ops.iou of one detection and one ground truth, both [y1, x1, y2, x2]
__device__ __forceinline__ double box_iou64(const double* d, const double* g) {
  const double ih = np_max(0.0, __dsub_rn(np_min(d[2], g[2]), np_max(d[0], g[0])));
  const double iw = np_max(0.0, __dsub_rn(np_min(d[3], g[3]), np_max(d[1], g[1])));
  const double inter = __dmul_rn(ih, iw);
  const double a1 = __dmul_rn(__dsub_rn(d[2], d[0]), __dsub_rn(d[3], d[1]));
  const double a2 = __dmul_rn(__dsub_rn(g[2], g[0]), __dsub_rn(g[3], g[1]));
  return __ddiv_rn(inter, __dsub_rn(__dadd_rn(a1, a2), inter));
}

// One thread per (image, class) segment of the segment order: greedy matching, 0 = FP, 1 = TP, 2 = beyond the 10,000.
__global__ void match_kernel(step_eval_rows R, int n, const unsigned long long* keys, const uint32_t* order,
                             const double* gt_box, const int* gt_cls, const int* gt_img_off, unsigned char* taken,
                             unsigned char* label) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || (j > 0 && keys[j] == keys[j - 1])) return;
  const unsigned long long key = keys[j];
  int end = j + 1;
  while (end < n && keys[end] == key) ++end;
  const int c = (int)(key >> 20), im = (int)(key & 0xfffff);
  int g0 = gt_img_off[im], g1 = gt_img_off[im + 1];
  while (g0 < g1 && gt_cls[g0] != c) ++g0;
  int ge = g0;
  while (ge < g1 && gt_cls[ge] == c) ++ge;
  const double4* boxes = reinterpret_cast<const double4*>(R.box);
  int seen = 0;
  for (int s = j; s < end;) {
    const int sc = R.scode[order[s]];
    int e = s + 1;
    while (e < end && R.scode[order[e]] == sc) ++e;
    for (int t = e - 1; t >= s; --t, ++seen) {  // equal scores: the later row first
      const uint32_t r = order[t];
      if (seen >= kMaxPerSegment) { label[r] = 2; continue; }
      unsigned char tp = 0;
      if (ge > g0) {
        const double4 b4 = boxes[r];
        const double d[4] = {b4.x, b4.y, b4.z, b4.w};
        int best = g0;
        double bv = 0.0;
        for (int g = g0; g < ge; ++g) {  // np.argmax: the first maximum, a NaN first of all
          const double v = box_iou64(d, gt_box + (size_t)g * 4);
          if (v != v) { best = g; bv = v; break; }
          if (g == g0 || v > bv) { best = g; bv = v; }
        }
        if (bv >= 0.5 && !taken[best]) { taken[best] = 1; tp = 1; }
      }
      label[r] = tp;
    }
    s = e;
  }
}

__global__ void class_bounds_kernel(step_eval_rows R, int n, const uint32_t* order, int* cls_start, int* cls_end) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int c = R.cls[order[j]];
  if (j == 0 || R.cls[order[j - 1]] != c) cls_start[c] = j;
  if (j == n - 1 || R.cls[order[j + 1]] != c) cls_end[c] = j + 1;
}

// numpy's pairwise sum of a[0, n) for 8 <= n <= 128 (eight partial sums), or n < 8 (in order)
__device__ double pairwise_leaf(const double* a, int n) {
  if (n < 8) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r = __dadd_rn(r, a[i]);
    return r;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, a[i]);
  return res;
}

__device__ __forceinline__ int pairwise_split(int n) { const int h = n / 2; return h - h % 8; }

// One CTA per class: precision / recall over the class order, the suffix maximum, the AP terms, their pairwise sum.
// Scratch of class c: prec and tpos at [s, e) of the class's rows, terms at [s + c, e + c + 1).
__global__ void __launch_bounds__(kApThreads) ap_kernel(int n_classes, const uint32_t* order, const unsigned char* label,
                                                         const int* cls_start, const int* cls_end, const int* num_gt,
                                                         double* prec, int* tpos, double* terms, double* ap) {
  const int c = blockIdx.x, tid = threadIdx.x;
  const int G = num_gt[c];
  if (G == 0) {
    if (tid == 0) ap[c] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const int s = cls_start[c], e = cls_end[c];
  __shared__ int s_kept, s_tp;
  __shared__ double s_carry;
  if (tid == 0) { s_kept = 0; s_tp = 0; s_carry = 0.0; }
  __syncthreads();
  // precision at every kept row, and the kept position of every TP
  for (int base = s; base < e; base += kApThreads) {
    const int j = base + tid;
    const int lab = j < e ? label[order[j]] : 2;
    int2 tot;
    const int2 inc = block_incl_scan2<kApThreads>(make_int2(lab != 2, lab == 1), &tot);
    if (lab != 2) {
      const int k = s_kept + inc.x - 1, ct = s_tp + inc.y;
      prec[s + k] = __ddiv_rn((double)ct, (double)(k + 1));
      if (lab == 1) tpos[s + ct - 1] = k;
    }
    __syncthreads();
    if (tid == 0) { s_kept += tot.x; s_tp += tot.y; }
    __syncthreads();
  }
  const int kept = s_kept, ntp = s_tp;
  if (kept == 0) {  // compute_average_precision of an empty precision array
    if (tid == 0) ap[c] = 0.0;
    return;
  }
  // precision[i] = max(precision[i], precision[i + 1]) from the end (the appended 0 changes nothing)
  __shared__ double wmax[kApThreads / 32];
  const int lane = tid & 31, w = tid >> 5;
  for (int top = kept; top > 0; top -= kApThreads) {
    const int idx = top - 1 - tid;
    double v = idx >= 0 ? prec[s + idx] : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v = fmax(v, u); }
    if (lane == 31) wmax[w] = v;
    __syncthreads();
    if (w == 0) {
      double t = wmax[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const double u = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t = fmax(t, u); }
      wmax[lane] = t;
    }
    __syncthreads();
    if (w > 0) v = fmax(v, wmax[w - 1]);
    v = fmax(v, s_carry);
    if (idx >= 0) prec[s + idx] = v;
    __syncthreads();
    if (tid == kApThreads - 1) s_carry = v;
    __syncthreads();
  }
  // (recall[i] - recall[i - 1]) * precision[i] at every recall change: each TP, then the end point while #TP < G
  double* T = terms + s + c;
  const double dG = (double)G;
  for (int t = tid; t < ntp; t += kApThreads)
    T[t] = __dmul_rn(__dsub_rn(__ddiv_rn((double)(t + 1), dG), __ddiv_rn((double)t, dG)), prec[s + tpos[s + t]]);
  const int nt = ntp + (ntp < G ? 1 : 0);
  if (tid == 0 && ntp < G) T[ntp] = __dmul_rn(__dsub_rn(1.0, __ddiv_rn((double)ntp, dG)), 0.0);
  __syncthreads();
  // np.sum: leaves of at most 128 terms, in parallel, then the tree from its leaves (prec / tpos are free now)
  int* leaf_start = tpos + s;
  double* leaf_sum = prec + s;
  __shared__ int s_leaves;
  if (tid == 0) {
    int stack[64][2], sp = 0, nl = 0;
    stack[sp][0] = 0; stack[sp][1] = nt; ++sp;
    while (sp) {
      --sp;
      const int a = stack[sp][0], m = stack[sp][1];
      if (m <= kPairwiseLeaf) { leaf_start[nl++] = a; continue; }
      const int h = pairwise_split(m);
      stack[sp][0] = a + h; stack[sp][1] = m - h; ++sp;  // right half visited after the left
      stack[sp][0] = a; stack[sp][1] = h; ++sp;
    }
    s_leaves = nl;
  }
  __syncthreads();
  const int nl = s_leaves;
  for (int l = tid; l < nl; l += kApThreads) {
    const int a = leaf_start[l], b = l + 1 < nl ? leaf_start[l + 1] : nt;
    leaf_sum[l] = pairwise_leaf(T + a, b - a);
  }
  __syncthreads();
  if (tid == 0) {
    // post-order walk of the same tree: a node's value is its left value plus its right value
    int stack[64][3], sp = 0, next_leaf = 0;  // (size, state, -) ; state 0: unvisited, 1: left done
    double vals[64];
    stack[sp][0] = nt; stack[sp][1] = 0; ++sp;
    double result = 0.0;
    while (sp) {
      int* top = stack[sp - 1];
      const int m = top[0];
      if (m <= kPairwiseLeaf) {
        double v = leaf_sum[next_leaf++];
        --sp;
        while (true) {  // hand v to the parent
          if (sp == 0) { result = v; break; }
          int* p = stack[sp - 1];
          if (p[1] == 0) {  // left child done: keep it, visit the right child
            vals[sp - 1] = v;
            p[1] = 1;
            const int h = pairwise_split(p[0]);
            stack[sp][0] = p[0] - h; stack[sp][1] = 0; ++sp;
            break;
          }
          v = __dadd_rn(vals[sp - 1], v);
          --sp;
        }
      } else {
        const int h = pairwise_split(m);
        stack[sp][0] = h; stack[sp][1] = 0; ++sp;
      }
    }
    ap[c] = __dadd_rn(0.0, result);
  }
}

// ---- workspace ----
struct EvalWs {
  size_t off[12];
  size_t bytes;
  EvalWs(int n, int n_classes, int n_gt) {
    const size_t nn = (size_t)(n > 0 ? n : 1), nb = (size_t)ceil_div(nn, kSortTile);
    const size_t sizes[12] = {nn * 8, nn * 8, nn * 4, nn * 4,    // keys, keys', vals, vals'
                              256 * nb * 4,                        // digit histograms
                              nn,                                  // labels
                              nn * 8, nn * 4,                      // precision, TP positions
                              (nn + (size_t)n_classes + 1) * 8,    // AP terms
                              (size_t)n_classes * 4, (size_t)n_classes * 4,  // class bounds
                              (size_t)(n_gt > 0 ? n_gt : 1)};      // taken flags
    size_t o = 0;
    for (int i = 0; i < 12; ++i) { off[i] = o; o += (sizes[i] + 255) & ~(size_t)255; }
    bytes = o;
  }
};

}  // namespace step

using namespace step;

static int eval_rows_check(const step_eval_rows* r, const char* who) {
  STEP_CHECK_ARG(r->capacity >= 0 && r->capacity <= STEP_EVAL_MAX_ROWS, "%s: rows.capacity %lld outside [0, %d]", who,
                 r->capacity, STEP_EVAL_MAX_ROWS);
  STEP_CHECK_ARG(r->counters && r->img_first, "%s: null pointer (rows.counters / rows.img_first)", who);
  STEP_CHECK_ARG(r->capacity == 0 || (r->box && r->score && r->scode && r->img && r->cls),
                 "%s: null pointer (rows.box / score / scode / img / cls)", who);
  return 0;
}

extern "C" int step_eval_append_check(const step_eval_append_params* p) {
  STEP_CHECK_ARG(p != nullptr, "eval_append: null params");
  STEP_CHECK_ARG(p->B >= 0 && p->B <= STEP_EVAL_MAX_CLIPS, "eval_append: B %d outside [0, %d]", p->B, STEP_EVAL_MAX_CLIPS);
  STEP_CHECK_ARG(p->cap >= 1 && p->ncls >= 1, "eval_append: bad cap %d / ncls %d", p->cap, p->ncls);
  STEP_CHECK_ARG((long long)p->B * p->cap <= STEP_EVAL_MAX_ROWS, "eval_append: B * cap %lld exceeds %d",
                 (long long)p->B * p->cap, STEP_EVAL_MAX_ROWS);
  STEP_CHECK_ARG(p->det && p->count && p->class_of, "eval_append: null pointer (det / count / class_of)");
  for (int b = 0; b < p->B; ++b)
    STEP_CHECK_ARG(p->img[b] >= -1 && p->img[b] < STEP_EVAL_MAX_IMAGES, "eval_append: img[%d] %d outside [-1, %d)", b,
                   p->img[b], STEP_EVAL_MAX_IMAGES);
  return eval_rows_check(&p->rows, "eval_append");
}

extern "C" int step_eval_append(const step_eval_append_params* p, step_stream_t stream) {
  const int rc = step_eval_append_check(p);
  if (rc) return rc;
  if (p->B == 0) return 0;
  eval_append_kernel<<<1, 1024, 0, cu(stream)>>>(*p);
  STEP_LAUNCH_CHECK("eval_append_kernel");
  return 0;
}

extern "C" size_t step_eval_workspace_bytes(int n_rows, int n_classes, int n_gt) {
  return EvalWs(n_rows, n_classes, n_gt).bytes;
}

extern "C" int step_eval_check(const step_eval_params* p) {
  STEP_CHECK_ARG(p != nullptr, "eval_run: null params");
  int rc = eval_rows_check(&p->rows, "eval_run");
  if (rc) return rc;
  STEP_CHECK_ARG(p->n_rows >= 0 && p->n_rows <= p->rows.capacity, "eval_run: n_rows %d outside [0, rows.capacity %lld]",
                 p->n_rows, p->rows.capacity);
  STEP_CHECK_ARG(p->n_classes >= 1 && p->n_classes <= STEP_EVAL_MAX_CLASSES, "eval_run: n_classes %d outside [1, %d]",
                 p->n_classes, STEP_EVAL_MAX_CLASSES);
  STEP_CHECK_ARG(p->n_images >= 0 && p->n_images <= STEP_EVAL_MAX_IMAGES, "eval_run: n_images %d outside [0, %d]", p->n_images,
                 STEP_EVAL_MAX_IMAGES);
  STEP_CHECK_ARG(p->n_gt >= 0 && p->max_gt_per_image >= 0 && p->max_gt_per_image <= STEP_EVAL_MAX_GT_PER_IMAGE,
                 "eval_run: n_gt %d / max_gt_per_image %d (at most %d ground-truth rows per image)", p->n_gt,
                 p->max_gt_per_image, STEP_EVAL_MAX_GT_PER_IMAGE);
  STEP_CHECK_ARG(p->gt_img_off && p->num_gt && p->ap && p->workspace, "eval_run: null pointer (gt_img_off / num_gt / ap / workspace)");
  STEP_CHECK_ARG(p->n_gt == 0 || (p->gt_box && p->gt_cls), "eval_run: null pointer (gt_box / gt_cls)");
  const size_t need = step_eval_workspace_bytes(p->n_rows, p->n_classes, p->n_gt);
  STEP_CHECK_ARG(p->workspace_bytes >= need, "eval_run: workspace_bytes %zu below the %zu needed", p->workspace_bytes, need);
  return 0;
}

extern "C" int step_eval_run(const step_eval_params* p, step_stream_t stream) {
  const int rc = step_eval_check(p);
  if (rc) return rc;
  const cudaStream_t st = cu(stream);
  const int n = p->n_rows;
  const EvalWs ws(n, p->n_classes, p->n_gt);
  unsigned char* w = static_cast<unsigned char*>(p->workspace);
  unsigned long long* k0 = (unsigned long long*)(w + ws.off[0]);
  unsigned long long* k1 = (unsigned long long*)(w + ws.off[1]);
  uint32_t* v0 = (uint32_t*)(w + ws.off[2]);
  uint32_t* v1 = (uint32_t*)(w + ws.off[3]);
  int* hist = (int*)(w + ws.off[4]);
  unsigned char* label = w + ws.off[5];
  double* prec = (double*)(w + ws.off[6]);
  int* tpos = (int*)(w + ws.off[7]);
  double* terms = (double*)(w + ws.off[8]);
  int* cls_start = (int*)(w + ws.off[9]);
  int* cls_end = (int*)(w + ws.off[10]);
  unsigned char* taken = w + ws.off[11];
  const int init_n = p->n_classes > p->n_gt ? p->n_classes : p->n_gt;
  eval_init_kernel<<<ceil_div(init_n > 0 ? init_n : 1, 256), 256, 0, st>>>(cls_start, cls_end, p->n_classes, taken, p->n_gt);
  STEP_LAUNCH_CHECK("eval_init_kernel");
  const uint32_t* order = v0;      // the class order
  if (n > 0) {
    const int g = ceil_div(n, 256);
    class_key_kernel<<<g, 256, 0, st>>>(p->rows, n, k0, v0);
    STEP_LAUNCH_CHECK("class_key_kernel");
    bool second;
    int r = radix_sort(k0, v0, k1, v1, n, 59, hist, st, &second);
    if (r) return r;
    // the class order is kept; the segment order is sorted in the other pair of buffers
    order = second ? v1 : v0;
    unsigned long long* sk = second ? k0 : k1;
    uint32_t* sv = second ? v0 : v1;
    unsigned long long* tk = second ? k1 : k0;  // scratch keys for the segment sort (the class keys are not needed)
    segment_key_kernel<<<g, 256, 0, st>>>(p->rows, n, order, sk, sv);
    STEP_LAUNCH_CHECK("segment_key_kernel");
    // a second value buffer is needed: reuse prec's bytes (8n >= 4n) until the matching is done
    uint32_t* sv2 = (uint32_t*)prec;
    r = radix_sort(sk, sv, tk, sv2, n, 27, hist, st, &second);
    if (r) return r;
    const unsigned long long* seg_keys = second ? tk : sk;
    const uint32_t* seg_order = second ? sv2 : sv;
    match_kernel<<<g, 256, 0, st>>>(p->rows, n, seg_keys, seg_order, p->gt_box, p->gt_cls, p->gt_img_off, taken, label);
    STEP_LAUNCH_CHECK("match_kernel");
    class_bounds_kernel<<<g, 256, 0, st>>>(p->rows, n, order, cls_start, cls_end);
    STEP_LAUNCH_CHECK("class_bounds_kernel");
  }
  ap_kernel<<<p->n_classes, kApThreads, 0, st>>>(p->n_classes, order, label, cls_start, cls_end, p->num_gt, prec, tpos, terms,
                                                 p->ap);
  STEP_LAUNCH_CHECK("ap_kernel");
  return 0;
}
