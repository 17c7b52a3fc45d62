// select.cu -- train_select (utils/utils.py:135-340) and select_proposals (:342-423) on the device, one refinement step
// per launch, with the reference's numpy and Python random draws made from device copies of the two MT19937 states.
//
// One CTA walks the clips in the reference's order (the draws are serial).  Per clip, the threads rank the candidates and
// compute the IoU; thread 0 assigns the positives and makes the draws; the threads then write the clip's rows.
// Arithmetic follows numpy's types: float32 operations are rounded one at a time (the file is built with -fmad=false),
// the choice weights and their cdf are float64.  Two parity contracts (README.md): every argsort(x)[::-1] is a
// stable ascending argsort reversed, and the softmax weights use the correctly rounded float32(exp(float64(x))).
// target_mode STEP_TARGETS_CLS writes the rows of train_cls.py:271-291 instead (step 1 only): same IoU, assignment and draws.
#include <limits.h>

#include "common.cuh"
#include "tube_math.cuh"

namespace step {

constexpr int kSelThreads = 256;
constexpr int kSelMaxSmem = 200 * 1024;  // below the 227 KB opt-in limit, which includes the kernel's static shared memory

// ---- MT19937, as numpy's legacy RandomState and CPython's random module run it ----
__device__ uint32_t mt_next(uint32_t* s) {
  int pos = (int)s[624];
  if (pos >= 624) {
    const uint32_t UP = 0x80000000u, LO = 0x7fffffffu, A = 0x9908b0dfu;
    int k = 0;
    for (; k < 624 - 397; ++k) {
      uint32_t y = (s[k] & UP) | (s[k + 1] & LO);
      s[k] = s[k + 397] ^ (y >> 1) ^ ((y & 1u) ? A : 0u);
    }
    for (; k < 623; ++k) {
      uint32_t y = (s[k] & UP) | (s[k + 1] & LO);
      s[k] = s[k + 397 - 624] ^ (y >> 1) ^ ((y & 1u) ? A : 0u);
    }
    uint32_t y = (s[623] & UP) | (s[0] & LO);
    s[623] = s[396] ^ (y >> 1) ^ ((y & 1u) ? A : 0u);
    pos = 0;
  }
  uint32_t y = s[pos];
  s[624] = (uint32_t)(pos + 1);
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// RandomState.random_sample: 53 bits from two outputs
__device__ double mt_double(uint32_t* s) {
  uint32_t a = mt_next(s) >> 5, b = mt_next(s) >> 6;
  return __ddiv_rn(__dadd_rn((double)a * 67108864.0, (double)b), 9007199254740992.0);
}

// random._randbelow(n) = getrandbits(n.bit_length()) until < n
__device__ int py_randbelow(uint32_t* s, int n) {
  int k = 32 - __clz(n);
  uint32_t r;
  do { r = mt_next(s) >> (32 - k); } while (r >= (uint32_t)n);
  return (int)r;
}

// np.sum of a float32 vector: numpy's pairwise summation (8 accumulators, blocks of 128)
__device__ float pairwise_sum(const float* a, int n) {
  if (n < 8) {
    float r = 0.0f;
    for (int i = 0; i < n; ++i) r = __fadd_rn(r, a[i]);
    return r;
  }
  if (n <= 128) {
    float r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[i + j]);
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, a[i]);
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return __fadd_rn(pairwise_sum(a, n2), pairwise_sum(a + n2, n - n2));
}

// RandomState.choice(n, size, replace=False, p=w): draw size - found doubles, zero the weights found so far, cdf =
// cumsum / its last element, searchsorted(side='right'), keep each new index at its first occurrence.  w is overwritten.
__device__ void np_choice(uint32_t* s, double* w, double* cdf, double* x, int n, int size, int* out) {
  int got = 0;
  while (got < size) {
    const int m = size - got;
    for (int k = 0; k < m; ++k) x[k] = mt_double(s);
    for (int k = 0; k < got; ++k) w[out[k]] = 0.0;
    double c = 0.0;
    for (int i = 0; i < n; ++i) { c = __dadd_rn(c, w[i]); cdf[i] = c; }
    const double total = cdf[n - 1];
    for (int i = 0; i < n; ++i) cdf[i] = __ddiv_rn(cdf[i], total);
    const int start = got;
    for (int k = 0; k < m; ++k) {
      int lo = 0, hi = n;  // first i with cdf[i] > x
      while (lo < hi) { int mid = (lo + hi) >> 1; if (cdf[mid] <= x[k]) lo = mid + 1; else hi = mid; }
      bool seen = false;
      for (int q = start; q < got; ++q) seen |= out[q] == lo;
      if (!seen) out[got++] = lo;
    }
  }
}

// A value of compute_box_iou (tube_utils.py:269-308) with its numpy type: float32 op float32 rounds to float32, anything
// with a float64 (float64 proposals at step 1) to float64.
struct Num { double v; bool d; };
__device__ __forceinline__ Num nf(float v) { return {(double)v, false}; }
__device__ __forceinline__ Num nadd(Num a, Num b) {
  return (a.d || b.d) ? Num{__dadd_rn(a.v, b.v), true} : Num{(double)__fadd_rn((float)a.v, (float)b.v), false};
}
__device__ __forceinline__ Num nsub(Num a, Num b) {
  return (a.d || b.d) ? Num{__dsub_rn(a.v, b.v), true} : Num{(double)__fsub_rn((float)a.v, (float)b.v), false};
}
__device__ __forceinline__ Num nmul(Num a, Num b) {
  return (a.d || b.d) ? Num{__dmul_rn(a.v, b.v), true} : Num{(double)__fmul_rn((float)a.v, (float)b.v), false};
}
__device__ __forceinline__ Num ndiv(Num a, Num b) {
  return (a.d || b.d) ? Num{__ddiv_rn(a.v, b.v), true} : Num{(double)__fdiv_rn((float)a.v, (float)b.v), false};
}

// compute_tube_iou at one frame: 0 when either box sums (sequentially, in its type) to 0
__device__ float box_iou(const Num* g, const Num* a) {
  Num sg = {0.0, g[0].d}, sa = {0.0, a[0].d};
  for (int k = 0; k < 4; ++k) { sg = nadd(sg, g[k]); sa = nadd(sa, a[k]); }
  if (sg.v == 0.0 || sa.v == 0.0) return 0.0f;
  Num x1 = a[0].v > g[0].v ? a[0] : g[0], y1 = a[1].v > g[1].v ? a[1] : g[1];   // Python max / min keep the operand
  Num x2 = a[2].v < g[2].v ? a[2] : g[2], y2 = a[3].v < g[3].v ? a[3] : g[3];
  Num w = nsub(x2, x1), h = nsub(y2, y1);
  if (w.v <= 0.0) w.v = 0.0;   // np.maximum(., 0.) (NaN stays)
  if (h.v <= 0.0) h.v = 0.0;
  const bool hit = w.v > 0.0 && h.v > 0.0;
  Num inter = hit ? nmul(w, h) : Num{0.0, false};
  Num uni = nadd(nmul(nsub(g[2], g[0]), nsub(g[3], g[1])), nmul(nsub(a[2], a[0]), nsub(a[3], a[1])));
  if (hit) uni = nsub(uni, inter);
  // a Python 0. over a typed union keeps the union's type
  Num r = hit ? ndiv(inter, uni) : ndiv(Num{0.0, uni.d}, uni);
  return (float)r.v;
}

// Shared-memory layout of one clip's work, the same on host and device.
struct SelLayout {
  int C, n, g, E, rows, L, Lout;
  size_t off[20];
  size_t bytes;
  __host__ __device__ SelLayout(int C_, int n_, int g_, int K_, int rows_, int L_, int Lout_)
      : C(C_), n(n_), g(g_), E(C_ * K_), rows(rows_), L(L_), Lout(Lout_) {
    size_t sizes[20] = {
        2 * STEP_SELECT_MT_WORDS * 4,         // 0 mt
        (size_t)C * n * 4,                    // 1 mean scores
        (size_t)E * 4, (size_t)E * 4,         // 2 entry score, 3 entry tube
        (size_t)E * 4,                        // 4 entry position
        (size_t)n * 4, (size_t)n * 4,         // 5 tube min position, 6 tube best score
        (size_t)n * 4, (size_t)n * 4,         // 7 candidate tube, 8 candidate score
        (size_t)g * n * 4, (size_t)g * n * 4, // 9 ious, 10 greedy scratch
        (size_t)n * 4,                        // 11 occupied
        (size_t)n * 4, (size_t)n * 4,         // 12 hit list, 13 free list
        (size_t)n * 8, (size_t)n * 8, (size_t)n * 8,  // 14 weights, 15 cdf, 16 uniforms
        (size_t)n * 4,                        // 17 chosen
        (size_t)rows * 8,                     // 18 pairs
        (size_t)rows * (L + Lout) * 4 * 4};   // 19 staging of the selected tubes
    size_t o = 0;
    for (int i = 0; i < 20; ++i) { off[i] = o; o += (sizes[i] + 15) & ~(size_t)15; }
    bytes = o;
  }
};

__global__ void __launch_bounds__(kSelThreads) select_step_kernel(step_select_params p, int K_max) {
  extern __shared__ __align__(16) unsigned char sm[];
  const int tid = threadIdx.x, C = p.C, L = p.L;
  SelLayout lay(C, p.n_max, p.g_max, K_max, p.max_rows, L, p.Lout);
  uint32_t* mt = (uint32_t*)(sm + lay.off[0]);
  float* msc = (float*)(sm + lay.off[1]);
  float* es = (float*)(sm + lay.off[2]);
  int* et = (int*)(sm + lay.off[3]);
  int* ep = (int*)(sm + lay.off[4]);
  int* minpos = (int*)(sm + lay.off[5]);
  float* best = (float*)(sm + lay.off[6]);
  int* ct = (int*)(sm + lay.off[7]);
  float* cs = (float*)(sm + lay.off[8]);
  float* iou = (float*)(sm + lay.off[9]);
  float* tmp = (float*)(sm + lay.off[10]);
  int* occ = (int*)(sm + lay.off[11]);
  int* hit = (int*)(sm + lay.off[12]);
  int* fre = (int*)(sm + lay.off[13]);
  double* w = (double*)(sm + lay.off[14]);
  double* cdf = (double*)(sm + lay.off[15]);
  double* xs = (double*)(sm + lay.off[16]);
  int* chosen = (int*)(sm + lay.off[17]);
  int2* pairs = (int2*)(sm + lay.off[18]);
  float* stage = (float*)(sm + lay.off[19]);
  __shared__ int s_nc, s_npos, s_rows, s_base;

  for (int i = tid; i < 2 * STEP_SELECT_MT_WORDS; i += blockDim.x) mt[i] = p.mt[i];
  if (tid == 0) s_base = 0;
  const int TC = 4 + C, OC = 6 + C;
  for (int b = 0; b < p.B; ++b) {
    const int off = p.tube_off[b], n = p.tube_off[b + 1] - off;
    const int g0 = p.gt_off[b], G = p.gt_off[b + 1] - g0;
    const float* tg = p.targets + (size_t)g0 * p.max_chunks * TC;
    __syncthreads();
    int Nc;
    if (p.step > 1) {
      // utils.py:177 torch.mean over the frames: sequential float32 sum, / L
      for (int i = tid; i < C * n; i += blockDim.x) {
        const int c = i / n, r = i - c * n;
        const float* q = p.prob + (off + r) * p.prob_sr + c * p.prob_sc;
        float s = 0.0f;
        for (int t = 0; t < L; ++t) s = __fadd_rn(s, q[t * p.prob_sl]);
        msc[i] = __fdiv_rn(s, (float)L);
      }
      for (int r = tid; r < n; r += blockDim.x) minpos[r] = INT_MAX;
      __syncthreads();
      // utils.py:183-196: the first K tubes of each class in descending order (equal scores: larger index first)
      const int K = p.topk > 0 ? min((p.topk / C) * 2, n) : n;
      for (int i = tid; i < C * n; i += blockDim.x) {
        const int c = i / n, r = i - c * n;
        const float s = msc[i];
        int rank = 0;
        for (int q = 0; q < n; ++q) { const float v = msc[c * n + q]; rank += (v > s) || (v == s && q > r); }
        if (rank < K) { es[c * K + rank] = s; et[c * K + rank] = r; }
      }
      __syncthreads();
      // utils.py:199-201: Python's stable sort by score, reversed; then the first entry of each tube (:202-207)
      const int E = C * K;
      for (int e = tid; e < E; e += blockDim.x) {
        const float s = es[e];
        int pos = 0;
        for (int q = 0; q < E; ++q) { const float v = es[q]; pos += (v > s) || (v == s && q > e); }
        ep[e] = pos;
        atomicMin(&minpos[et[e]], pos);
      }
      __syncthreads();
      for (int e = tid; e < E; e += blockDim.x)
        if (ep[e] == minpos[et[e]]) best[et[e]] = es[e];
      __syncthreads();
      for (int r = tid; r < n; r += blockDim.x) {
        if (minpos[r] == INT_MAX) continue;
        int rank = 0;
        for (int q = 0; q < n; ++q) rank += minpos[q] < minpos[r];
        if (p.topk <= 0 || rank < p.topk) { ct[rank] = r; cs[rank] = best[r]; }
      }
      if (tid == 0) {
        int present = 0;
        for (int r = 0; r < n; ++r) present += minpos[r] != INT_MAX;
        s_nc = p.topk > 0 ? min(present, p.topk) : present;
      }
      __syncthreads();
      Nc = s_nc;
    } else {
      for (int r = tid; r < n; r += blockDim.x) ct[r] = r;
      Nc = n;
      __syncthreads();  // the IoU below reads every ct[j]
    }
    // select_proposals:348, the IoU of each ground truth's centre chunk and each candidate's centre frame
    for (int i = tid; i < G * Nc; i += blockDim.x) {
      const int g = i / Nc, j = i - g * Nc;
      Num gb[4], ab[4];
      for (int k = 0; k < 4; ++k) gb[k] = nf(tg[((size_t)g * p.max_chunks + p.gt_mid) * TC + k]);
      const size_t row = ((size_t)(off + ct[j]) * L + L / 2) * 4;
      if (p.step > 1) {
        float4 v = valid_one(ld4(p.loc + row), p.width, p.height);
        ab[0] = nf(v.x); ab[1] = nf(v.y); ab[2] = nf(v.z); ab[3] = nf(v.w);
      } else {
        for (int k = 0; k < 4; ++k) ab[k] = p.prop_f64 ? Num{p.props[row + k], true} : nf((float)p.props[row + k]);
      }
      iou[i] = box_iou(gb, ab);
      tmp[i] = iou[i];
    }
    __syncthreads();
    if (p.step == 1)  // select_proposals:349-350, scores = max IoU over the ground truths
      for (int j = tid; j < Nc; j += blockDim.x) {
        float m = iou[j];
        for (int g = 1; g < G; ++g) m = fmaxf(m, iou[g * Nc + j]);
        cs[j] = m;
      }
    __syncthreads();
    if (tid == 0) {
      uint32_t* np_mt = mt;
      uint32_t* py_mt = mt + STEP_SELECT_MT_WORDS;
      for (int j = 0; j < Nc; ++j) occ[j] = 0;
      int npos = 0;
      // :360-368, each ground truth in turn (the one with the largest remaining IoU) takes its best unoccupied candidate
      for (int it = 0; it < G; ++it) {
        int gi = 0;
        float gm = -INFINITY;
        for (int g = 0; g < G; ++g) {
          float m = tmp[g * Nc];
          for (int j = 1; j < Nc; ++j) m = fmaxf(m, tmp[g * Nc + j]);
          if (g == 0 || m > gm) { gm = m; gi = g; }
        }
        int bj = -1;
        for (int j = 0; j < Nc; ++j)
          if (!occ[j] && (bj < 0 || iou[gi * Nc + j] >= iou[gi * Nc + bj])) bj = j;
        if (bj >= 0) {
          occ[bj] = 1;
          pairs[npos++] = make_int2(gi, bj);
          for (int j = 0; j < Nc; ++j) tmp[gi * Nc + j] = -1.0f;
        }
      }
      // :369-371 (the pairs beyond max_pos only exist here, in this scratch list: max_rows bounds the output)
      if (npos > p.max_pos) {
        for (int i = npos - 1; i >= 1; --i) {
          int j = py_randbelow(py_mt, i + 1);
          int2 t = pairs[i]; pairs[i] = pairs[j]; pairs[j] = t;
        }
        npos = p.max_pos;
      }
      // :373-390, the other candidates above cls_thresh, drawn uniformly
      int nh = 0;
      for (int j = 0; j < Nc; ++j) {
        bool above = false;
        for (int g = 0; g < G; ++g) above |= iou[g * Nc + j] > p.cls_thresh;
        if (above && !occ[j]) hit[nh++] = j;
      }
      if (nh > 0 && npos < p.max_pos) {
        const int size = min(nh, p.max_pos - npos);
        for (int k = 0; k < nh; ++k) w[k] = 1.0 / (double)nh;
        np_choice(np_mt, w, cdf, xs, nh, size, chosen);
        for (int k = 0; k < size; ++k) {
          const int j = hit[chosen[k]];
          int gi = 0;
          for (int g = 1; g < G; ++g) if (iou[g * Nc + j] > iou[gi * Nc + j]) gi = g;
          occ[j] = 1;
          pairs[npos++] = make_int2(gi, j);
        }
      }
      for (int k = 0; k < nh; ++k) occ[hit[k]] = 1;
      // :398-417, negatives weighted by their scores
      int nf_ = 0;
      for (int j = 0; j < Nc; ++j) if (!occ[j]) fre[nf_++] = j;
      int rows = npos;
      const int size = min(npos * p.neg_ratio, nf_);
      if (size > 0) {
        float* a = (float*)xs;  // float32 weights before the float64 conversion (xs is free until the draw)
        if (p.sampling == STEP_SAMPLING_RANDOM) {
          for (int k = 0; k < nf_; ++k) w[k] = 1.0 / (double)nf_;
        } else {
          for (int k = 0; k < nf_; ++k) {
            const float s = cs[fre[k]];
            a[k] = p.sampling == STEP_SAMPLING_UNIFORM ? __fadd_rn(s, 1e-6f) : (float)exp((double)s);
          }
          const float tot = pairwise_sum(a, nf_);
          for (int k = 0; k < nf_; ++k) w[k] = (double)__fdiv_rn(a[k], tot);
        }
        np_choice(np_mt, w, cdf, xs, nf_, size, chosen);
        for (int k = 0; k < size; ++k) {
          const int j = fre[chosen[k]];
          int gi = 0;
          for (int g = 1; g < G; ++g) if (iou[g * Nc + j] > iou[gi * Nc + j]) gi = g;
          pairs[rows++] = make_int2(gi, j);
        }
      }
      s_npos = npos;
      s_rows = rows;
      p.counts[b] = rows;
    }
    __syncthreads();
    // utils.py:259-338: the selected rows at this clip's offset in the flat outputs
    const int npos = s_npos, rows = s_rows, base = s_base;
    const int T = p.T, Lout = p.Lout;
    for (int r = tid; r < rows; r += blockDim.x) {
      const int j = pairs[r].y, tube = off + ct[j];
      float* in = stage + (size_t)r * (L + Lout) * 4;
      float* ext = in + L * 4;
      for (int t = 0; t < L; ++t) {
        const size_t q = ((size_t)tube * L + t) * 4;
        float4 v;
        if (p.step > 1) v = valid_one(ld4(p.loc + q), p.width, p.height);
        else v = make_float4((float)p.props[q], (float)p.props[q + 1], (float)p.props[q + 2], (float)p.props[q + 3]);
        st4(in + t * 4, v);
      }
      if (p.ext_mode == STEP_EXT_NONE) {
        for (int t = 0; t < L * 4; ++t) ext[t] = in[t];
      } else if (p.ext_mode == STEP_EXT_PREDICT) {
        for (int t = 0; t < T; ++t) {
          st4(ext + t * 4, valid_one(ld4(p.first + ((size_t)tube * T + t) * 4), p.width, p.height));
          st4(ext + (T + L + t) * 4, valid_one(ld4(p.last + ((size_t)tube * T + t) * 4), p.width, p.height));
        }
        for (int t = 0; t < L * 4; ++t) ext[T * 4 + t] = in[t];
      } else if (p.ext_mode == STEP_EXT_EXTRAPOLATE) {
        for (int c = 0; c < 4; ++c) extrapolate_one(in, L, T, 400.0f, 400.0f, ext, c);  // its default 400 x 400 clamp
      } else {
        for (int c = 0; c < 4; ++c) {
          float s = 0.0f;
          for (int t = 0; t < L; ++t) s = __fadd_rn(s, in[t * 4 + c]);
          const float m = __fdiv_rn(s, (float)L);
          for (int t = 0; t < T; ++t) { ext[t * 4 + c] = m; ext[(T + L + t) * 4 + c] = m; }
          for (int t = 0; t < L; ++t) ext[(T + t) * 4 + c] = in[t * 4 + c];
        }
      }
      float* o = p.out_tubes + (size_t)(base + r) * Lout * 5;
      for (int t = 0; t < Lout; ++t) {   // flatten_tubes(batch_idx=True): arange(Lout) + b * Lout first
        o[t * 5] = (float)(b * Lout + t);
        for (int c = 0; c < 4; ++c) o[t * 5 + 1 + c] = ext[t * 4 + c];
      }
    }
    for (int i = tid; i < rows * 3 * OC; i += blockDim.x) {
      const int r = i / (3 * OC), k = (i / OC) % 3, col = i % OC;
      const int g = pairs[r].x, j = pairs[r].y;
      const bool pos = r < npos;
      float v = 0.0f;
      if (p.target_mode == STEP_TARGETS_CLS) {   // train_cls.py:274-288: one centre row, copied to all three
        const float* src = tg + ((size_t)g * p.max_chunks + p.gt_mid) * TC;
        v = col == 4 ? 1.0f : col == 5 || !pos ? 0.0f : col < 4 ? src[col] : src[col - 2];
      } else if (k == 1) {
        if (pos || iou[g * Nc + j] >= p.reg_thresh) {
          const float* src = tg + ((size_t)g * p.max_chunks + p.gt_mid) * TC;
          v = col < 4 ? src[col] : col == 4 ? (pos ? 1.0f : 0.0f) : col == 5 ? 1.0f : src[col - 2];
        }
      } else if (p.predict_nb && pos) {
        const float* src = tg + ((size_t)g * p.max_chunks + (k == 0 ? p.nb_first : p.nb_last)) * TC;
        if (col < 4) v = src[col];
        else if (col == 5) v = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.0f, src[0]), src[1]), src[2]), src[3]) > 0.0f ? 1.0f : 0.0f;
        else if (col > 5) v = src[col - 2];
      }
      p.out_targets[(size_t)(base + r) * 3 * OC + k * OC + col] = v;
    }
    __syncthreads();
    if (tid == 0) s_base = base + rows;
  }
  __syncthreads();
  for (int i = tid; i < 2 * STEP_SELECT_MT_WORDS; i += blockDim.x) p.mt[i] = mt[i];
}

}  // namespace step

using namespace step;

// Every check that needs no pointer, and the kernel's shared memory: K (entries per class) and the scratch pair count.
static int select_check_fields(const step_select_params* p, int* K_out, int* pairs_out, size_t* smem_out) {
  STEP_CHECK_ARG(p != nullptr, "select_step: null params");
  STEP_CHECK_ARG(p->step >= 1 && p->B >= 1 && p->C >= 1 && p->L >= 1 && p->T >= 1,
                 "select_step: bad step %d / B %d / C %d / L %d / T %d", p->step, p->B, p->C, p->L, p->T);
  STEP_CHECK_ARG(p->ext_mode >= STEP_EXT_NONE && p->ext_mode <= STEP_EXT_MEAN, "select_step: bad ext_mode %d", p->ext_mode);
  STEP_CHECK_ARG(p->step > 1 || p->ext_mode == STEP_EXT_NONE, "select_step: step 1 has no previous chunk count to extend from");
  STEP_CHECK_ARG(p->Lout == p->L + (p->ext_mode != STEP_EXT_NONE ? 2 * p->T : 0),
                 "select_step: T_length %d does not match L=%d, T=%d and ext_mode %d", p->Lout, p->L, p->T, p->ext_mode);
  STEP_CHECK_ARG(p->ext_mode != STEP_EXT_EXTRAPOLATE || (p->T >= 2 && p->L >= p->T), "select_step: EXTRAPOLATE needs L >= T >= 2");
  STEP_CHECK_ARG(p->target_mode == STEP_TARGETS_SELECT || p->target_mode == STEP_TARGETS_CLS, "select_step: bad target_mode %d",
                 p->target_mode);
  STEP_CHECK_ARG(p->target_mode != STEP_TARGETS_CLS || (p->step == 1 && p->ext_mode == STEP_EXT_NONE && !p->predict_nb),
                 "select_step: target_mode %d needs step 1, no extension and no neighbour rows (step %d, ext_mode %d, "
                 "predict_nb %d)", p->target_mode, p->step, p->ext_mode, p->predict_nb);
  STEP_CHECK_ARG(p->max_chunks >= 1 && p->gt_mid >= 0 && p->gt_mid < p->max_chunks, "select_step: gt_mid %d outside %d chunks",
                 p->gt_mid, p->max_chunks);
  STEP_CHECK_ARG(!p->predict_nb || (p->nb_first >= 0 && p->nb_first < p->max_chunks && p->nb_last >= 0 && p->nb_last < p->max_chunks),
                 "select_step: neighbour chunks %d / %d outside %d chunks", p->nb_first, p->nb_last, p->max_chunks);
  STEP_CHECK_ARG(!(p->topk > 0 && p->topk < p->C), "select_step: 0 < topk=%d < C=%d keeps no candidate", p->topk, p->C);
  STEP_CHECK_ARG(p->max_pos >= 0 && p->neg_ratio >= 0, "select_step: bad max_pos %d / neg_ratio %d", p->max_pos, p->neg_ratio);
  STEP_CHECK_ARG(p->sampling >= STEP_SAMPLING_UNIFORM && p->sampling <= STEP_SAMPLING_SOFTMAX, "select_step: bad sampling %d",
                 p->sampling);
  STEP_CHECK_ARG(p->max_rows >= 0 && (long long)p->max_pos * (1 + p->neg_ratio) <= p->max_rows,
                 "select_step: max_pos %d * (1 + neg_ratio %d) rows exceed max_rows %d", p->max_pos, p->neg_ratio, p->max_rows);
  STEP_CHECK_ARG(p->n_max >= 1 && p->g_max >= 1, "select_step: bad n_max %d / g_max %d", p->n_max, p->g_max);
  const int K = p->step > 1 && p->topk > 0 ? (p->topk / p->C * 2 < p->n_max ? p->topk / p->C * 2 : p->n_max) : p->n_max;
  const int rows = p->max_pos + p->max_pos * p->neg_ratio;   // rows a clip can produce, before the shuffle's cut
  const int pairs = rows > p->g_max + p->n_max ? rows : p->g_max + p->n_max;
  SelLayout lay(p->C, p->n_max, p->g_max, p->step > 1 ? K : 0, pairs, p->L, p->Lout);
  STEP_CHECK_ARG(lay.bytes <= (size_t)kSelMaxSmem, "select_step: %zu bytes of shared memory for n_max %d, g_max %d, C %d exceed %d",
                 lay.bytes, p->n_max, p->g_max, p->C, kSelMaxSmem);
  *K_out = p->step > 1 ? K : 0;
  *pairs_out = pairs;
  *smem_out = lay.bytes;
  return 0;
}

extern "C" int step_select_check_f32(const step_select_params* p) {
  int K, pairs;
  size_t smem;
  return select_check_fields(p, &K, &pairs, &smem);
}

extern "C" int step_select_step_f32(const step_select_params* p, step_stream_t stream) {
  int K, pairs;
  size_t smem;
  int rc = select_check_fields(p, &K, &pairs, &smem);
  if (rc) return rc;
  STEP_CHECK_ARG(p->tube_off && p->gt_off && p->targets && p->mt && p->out_tubes && p->out_targets && p->counts,
                 "select_step: null pointer");
  STEP_CHECK_ARG(p->step > 1 || p->props, "select_step: null pointer (props)");
  STEP_CHECK_ARG(p->step == 1 || (p->prob && p->loc), "select_step: null pointer (prob / loc)");
  STEP_CHECK_ARG(p->ext_mode != STEP_EXT_PREDICT || (p->first && p->last), "select_step: null pointer (first / last)");
  static std::atomic<unsigned long long> seen{0};
  rc = allow_dynamic_smem(select_step_kernel, seen, kSelMaxSmem, "select_step");
  if (rc) return rc;
  step_select_params q = *p;
  q.max_rows = pairs;  // the kernel's scratch pair list; the output rows stay within p->max_rows
  select_step_kernel<<<1, kSelThreads, smem, cu(stream)>>>(q, K);
  STEP_LAUNCH_CHECK("select_step_kernel");
  return 0;
}
