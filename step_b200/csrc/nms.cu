// nms.cu -- bit-exact greedy NMS on sm_90a, fully device resident.
//
// Replaces _C.nms (external/maskrcnn_benchmark/csrc/nms.h:34-51).  The semantics every reference
// driver exercises are the CPU ones (test.py:192 calls nms on CPU tensors): legacy "+1" areas,
// suppress when IoU >= thr (cpu/nms_cpu.cpp:84); ge=0 gives the CUDA variant (cuda/nms.cu:84, '>').
// The IoU predicate is evaluated with explicitly rounded fp32 operations (__fadd_rn/__fmul_rn/
// __fdiv_rn: no FMA contraction, IEEE division) in the operand order of nms_cpu.cpp:74-83 so the
// keep set is bit-identical to the reference's.  Unlike cuda/nms.cu:118-147 there is no blocking
// D2H copy and no host scan: ordering, the 64x64 bitmask tiles, the greedy resolve and the
// compaction all run on the caller's stream.
#include "common.cuh"
#include "tube_math.cuh"

namespace step {

__device__ __forceinline__ float box_area(float4 b) {
  // nms_cpu.cpp:46  (x2 - x1 + 1) * (y2 - y1 + 1)
  return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
}

// std::max(p, q) is (p < q) ? q : p and std::min(p, q) is (q < p) ? q : p: a NaN p is returned, a NaN q is dropped, and
// p is returned when the two are equal (+0.0 against -0.0).  Python's builtin max / min follow the same rule.
__device__ __forceinline__ float std_max(float p, float q) { return (p < q) ? q : p; }
__device__ __forceinline__ float std_min(float p, float q) { return (q < p) ? q : p; }

__device__ __forceinline__ bool suppresses(float4 a, float area_a, float4 b, float area_b, float thr, int ge) {
  // nms_cpu.cpp:74-85, a the earlier row (ix1...), b the later one (x1[j]...)
  float xx1 = std_max(a.x, b.x), yy1 = std_max(a.y, b.y);
  float xx2 = std_min(a.z, b.z), yy2 = std_min(a.w, b.w);
  float w = std_max(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
  float h = std_max(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
  float inter = __fmul_rn(w, h);
  float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
  return ge ? (ovr >= thr) : (ovr > thr);
}

// ---- 1. ordering: rank sort (score desc, index asc).  O(n^2) compares, embarrassingly parallel;
//         10k boxes = 1e8 compares ~ 10 us.  Deterministic and stable by construction, unlike the
//         reference's torch.sort (unstable on ties).  NaN scores rank above every number, as
//         scores.sort(0, descending=True) (nms_cpu.cpp:48) puts them first, and -0.0 ties with +0.0.  The compares run on
//         order_key(score), an int with the same order, so every row gets a distinct rank: a float compare is false for
//         every NaN, which would give all NaN rows and the best row rank 0 and leave slots of `order` unwritten.
__device__ __forceinline__ int order_key(float s) {
  if (s != s) return 0x7fffffff;                     // NaN: above +inf (0x7f800000)
  const int b = __float_as_int(s == 0.0f ? 0.0f : s);  // -0.0 -> +0.0
  return b >= 0 ? b : b ^ 0x7fffffff;                // negatives: larger magnitude -> smaller key
}

__global__ void __launch_bounds__(256) nms_rank_kernel(const float* __restrict__ boxes,
                                                       const float* __restrict__ scores, int n,
                                                       float4* __restrict__ sorted_boxes,
                                                       int* __restrict__ order) {
  __shared__ int tile[1024];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int si = i < n ? order_key(scores[i]) : 0;
  int rank = 0;
  for (int base = 0; base < n; base += 1024) {
    int cnt = min(1024, n - base);
    for (int t = threadIdx.x; t < cnt; t += blockDim.x) tile[t] = order_key(scores[base + t]);
    __syncthreads();
    if (i < n) {
      // elements before i in index order win ties; split the loop so the compare is branch-free
      int lim = min(max(i - base, 0), cnt);
      for (int t = 0; t < lim; ++t) rank += (tile[t] >= si);
      for (int t = lim; t < cnt; ++t) rank += (tile[t] > si);
    }
    __syncthreads();
  }
  if (i < n) {
    sorted_boxes[rank] = reinterpret_cast<const float4*>(boxes)[i];
    order[rank] = i;
  }
}

// The pairwise predicates of the two greedy passes of this file.  prep(b) is the per-box value the predicate reuses (an
// area); p(a, prep(a), b, prep(b)) says whether the earlier box a takes the later box b.
struct NmsPred {   // nms_cpu.cpp:74-85: suppress when IoU >= thr (ge) or > thr, legacy "+1" areas
  float thr;
  int ge;
  __device__ __forceinline__ float prep(float4 b) const { return box_area(b); }
  __device__ __forceinline__ bool operator()(float4 a, float aa, float4 b, float ab) const {
    return suppresses(a, aa, b, ab, thr, ge);
  }
};

struct MergePred {  // demo.py:190  compute_box_iou(box, box2) > global_thresh  (utils/tube_utils.py:292-306, float32)
  float thr;
  __device__ __forceinline__ float prep(float4 b) const { return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y)); }
  __device__ __forceinline__ bool operator()(float4 a, float aa, float4 b, float ab) const {
    // Python's max / min on the coordinates (tube_utils.py:292-295), np.maximum(v, 0.) on the sides (NaN kept)
    const float iw = clamp_lo(__fsub_rn(std_min(a.z, b.z), std_max(a.x, b.x)), 0.0f);
    const float ih = clamp_lo(__fsub_rn(std_min(a.w, b.w), std_max(a.y, b.y)), 0.0f);
    const float inter = (iw > 0.0f && ih > 0.0f) ? __fmul_rn(iw, ih) : 0.0f;
    // a zero union gives NaN (two identical zero-area boxes), which never merges
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter)) > thr;
  }
};

// Where the greedy passes read their rows: count(z) rows of problem z (blockIdx.z of the mask pass, blockIdx.x of the
// resolve), box(z, i) the i-th in greedy order.
struct SortedRows {   // step_nms_f32: one problem, boxes already in score order
  const float4* sb;
  int n;
  __device__ __forceinline__ int count(int) const { return n; }
  __device__ __forceinline__ float4 box(int, int i) const { return sb[i]; }
};

struct DetRows {      // step_detect_merge_f32: clip z's rows det[z][0, det_count[z]) in step_detect_f32's order
  const float* det;
  const int* det_count;
  int cap;
  __device__ __forceinline__ int count(int z) const { return min(max(det_count[z], 0), cap); }
  __device__ __forceinline__ float4 box(int z, int i) const {
    return *reinterpret_cast<const float4*>(det + ((size_t)z * cap + i) * 8);
  }
};

// ---- 2. upper-triangular 64x64 bitmask tiles: bit j of mask[r][col_blk] = pred(row r, row col_blk*64 + j), j > r.
//         Problem z's mask starts at mask + z * mask_stride, col_blocks words per row.
constexpr int kTile = 64;
template <class Rows, class Pred>
__global__ void __launch_bounds__(kTile) mask_tiles_kernel(Rows rows, Pred pred, int col_blocks, size_t mask_stride,
                                                           unsigned long long* __restrict__ mask) {
  const int z = blockIdx.z, n = rows.count(z);
  const int row_blk = blockIdx.y, col_blk = blockIdx.x;
  if (col_blk < row_blk || col_blk * kTile >= n) return;  // never read by the resolve
  mask += (size_t)z * mask_stride;
  __shared__ float4 cb[kTile];
  __shared__ float ca[kTile];
  const int col_size = min(n - col_blk * kTile, kTile);
  if (threadIdx.x < col_size) {
    float4 b = rows.box(z, col_blk * kTile + threadIdx.x);
    cb[threadIdx.x] = b;
    ca[threadIdx.x] = pred.prep(b);
  }
  __syncthreads();
  const int r = row_blk * kTile + threadIdx.x;
  if (r < n) {
    float4 a = rows.box(z, r);
    float aa = pred.prep(a);
    unsigned long long bits = 0;
    int start = (row_blk == col_blk) ? threadIdx.x + 1 : 0;
    for (int j = start; j < col_size; ++j)
      if (pred(a, aa, cb[j], ca[j])) bits |= 1ULL << j;
    mask[(size_t)r * col_blocks + col_blk] = bits;
  }
}

// ---- 3. greedy resolve on device: one CTA per problem walks its 64-row blocks in order.  A row is kept (a leader) unless
//         an earlier kept row took it.  keep(z, i, k) stores row i's flag; claim(z, leader, col_blk, bits) is told which
//         rows of column block col_blk the kept row `leader` is the first to take (leaders are visited in ascending order).
struct KeepByOrder {  // step_nms_f32: flag at the row's original index
  const int* order;
  uint8_t* keep_flag;
  __device__ __forceinline__ void operator()(int, int i, unsigned k) const { keep_flag[order[i]] = (uint8_t)k; }
};

struct NoClaim {
  __device__ __forceinline__ void operator()(int, int, int, unsigned long long) const {}
};

template <class Rows, class Keep, class Claim>
__global__ void __launch_bounds__(1024) resolve_kernel(const unsigned long long* __restrict__ mask, Rows rows,
                                                       int col_ld, size_t mask_stride, Keep keep, Claim claim) {
  extern __shared__ unsigned long long remv[];  // [col_ld]
  __shared__ unsigned long long diag[kTile];
  __shared__ unsigned long long kept_s;
  const int z = blockIdx.x, n = rows.count(z), col_blocks = (n + kTile - 1) / kTile;
  mask += (size_t)z * mask_stride;
  for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) remv[j] = 0;
  __syncthreads();
  for (int blk = 0; blk < col_blocks; ++blk) {
    const int cnt = min(kTile, n - blk * kTile);
    if (threadIdx.x < cnt) diag[threadIdx.x] = mask[(size_t)(blk * kTile + threadIdx.x) * col_ld + blk];
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long r = remv[blk], kept = 0;
      for (int b = 0; b < cnt; ++b)
        if (!((r >> b) & 1ULL)) {
          kept |= 1ULL << b;
          claim(z, blk * kTile + b, blk, diag[b] & ~r);
          r |= diag[b];
        }
      kept_s = kept;
    }
    __syncthreads();
    const unsigned long long kept = kept_s;
    if (threadIdx.x < cnt) keep(z, blk * kTile + threadIdx.x, (unsigned)((kept >> threadIdx.x) & 1ULL));
    for (int j = blk + 1 + threadIdx.x; j < col_blocks; j += blockDim.x) {
      unsigned long long acc = remv[j], k = kept;
      while (k) {
        int b = __ffsll((long long)k) - 1;
        k &= k - 1;
        const unsigned long long m = mask[(size_t)(blk * kTile + b) * col_ld + j];
        claim(z, blk * kTile + b, j, m & ~acc);
        acc |= m;
      }
      remv[j] = acc;
    }
    __syncthreads();
  }
}

// Block-wide compaction in index order with a warp-ballot scan: calls emit(i, slot) for every i in [0, n) with flag(i)
// nonzero, slot = the number of such i before it, and returns their count.  Called by the whole CTA of kWarps warps.
template <int kWarps, class Flag, class Emit>
__device__ __forceinline__ int ballot_compact(int n, Flag flag, Emit emit) {
  __shared__ int warp_tot[kWarps];
  __shared__ int base_s;
  if (threadIdx.x == 0) base_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int start = 0; start < n; start += blockDim.x) {
    const int i = start + threadIdx.x;
    const int f = (i < n) ? flag(i) : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_tot[wid] = __popc(bal);
    __syncthreads();
    int off = base_s;
    for (int w = 0; w < wid; ++w) off += warp_tot[w];
    if (f) emit(i, off + __popc(bal & ((1u << lane) - 1)));
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < kWarps; ++w) t += warp_tot[w];
      base_s += t;
    }
    __syncthreads();
  }
  return base_s;
}

// ---- 4. compaction: kept original indices ascending (nms_cpu.cpp:88 nonzero(suppressed == 0))
__global__ void __launch_bounds__(1024) nms_compact_kernel(const uint8_t* __restrict__ keep_flag, int n,
                                                           int64_t* __restrict__ keep_out,
                                                           int* __restrict__ n_keep) {
  const int total = ballot_compact<32>(n, [&](int i) { return (int)keep_flag[i]; },
                                       [&](int i, int slot) { keep_out[slot] = i; });
  if (threadIdx.x == 0) *n_keep = total;
}

// ---- greedy NMS of one small problem in shared memory (nms_cpu.cpp:57-88), one CTA.  Rows i in [0, n) whose score
//      passes the threshold are ranked (score descending, index ascending), then suppressed in rank order; the other rows
//      are dropped.  Both callers' thresholds are ordered compares, so a NaN score never passes: it is dropped, as
//      scores.gt(conf_thresh) drops it in test.py:180.  The caller says how rows are read and where their keep flags go:
//        score(i)    row i's score;
//        pass(s)     whether a row of score s takes part;
//        box(i, s)   row i's box, asked once for every row before its threshold test;
//        keep(i, k)  stores row i's keep flag k.
constexpr int kSegMax = 1024;
template <class Score, class Pass, class Box, class Keep>
__device__ __forceinline__ void greedy_nms_smem(int n, float thr, int ge, Score score, Pass pass, Box box, Keep keep) {
  __shared__ float4 sb[kSegMax];
  __shared__ float sa[kSegMax];
  __shared__ float ss[kSegMax];
  __shared__ short sorig[kSegMax];
  __shared__ uint8_t sup[kSegMax];
  __shared__ int m_s;
  if (n <= 0) return;
  // the host bounds n (step_nms_segmented_max_rows(), step_detect_f32's max_per_clip); never overrun shared memory
  if (n > kSegMax) __trap();
  if (threadIdx.x == 0) m_s = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) ss[i] = score(i);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float si = ss[i];
    const float4 b = box(i, si);
    if (pass(si)) {
      int rank = 0;
      for (int t = 0; t < n; ++t) {
        const float st = ss[t];
        rank += pass(st) && ((st > si) || (st == si && t < i));
      }
      sb[rank] = b;
      sa[rank] = box_area(b);
      sorig[rank] = (short)i;
      atomicAdd(&m_s, 1);
    } else {
      keep(i, 0);
    }
  }
  __syncthreads();
  const int m = m_s;
  for (int i = threadIdx.x; i < m; i += blockDim.x) sup[i] = 0;
  __syncthreads();
  for (int i = 0; i < m; ++i) {
    if (!sup[i]) {  // uniform across the CTA (smem, synced)
      const float4 a = sb[i];
      const float aa = sa[i];
      for (int j = i + 1 + threadIdx.x; j < m; j += blockDim.x)
        if (!sup[j] && suppresses(a, aa, sb[j], sa[j], thr, ge)) sup[j] = 1;
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < m; i += blockDim.x) keep(sorig[i], sup[i] ? 0 : 1);
}

// ---- segmented small-problem kernel: one CTA per (clip, class) segment.
__global__ void __launch_bounds__(256) nms_segmented_kernel(const float* __restrict__ boxes,
                                                            const float* __restrict__ scores,
                                                            const int* __restrict__ seg_offsets, float thr,
                                                            int ge, float min_score,
                                                            uint8_t* __restrict__ keep_mask) {
  const int beg = seg_offsets[blockIdx.x], n = seg_offsets[blockIdx.x + 1] - beg;
  greedy_nms_smem(
      n, thr, ge, [&](int i) { return scores[beg + i]; },
      [&](float s) { return s >= min_score; },   // the confidence threshold of test.py:180 (false for NaN)
      [&](int i, float) { return reinterpret_cast<const float4*>(boxes)[beg + i]; },
      [&](int i, uint8_t k) { keep_mask[beg + i] = k; });
}


// ---- detection post-processing (test.py:156-218 / demo.py:121-198) -----------------------------------------------
// The reference drivers loop on the host over clips x classes: scores.gt(conf) -> valid_tubes(default 400x400) -> nms
// -> normalise -> (optional) the topk best scores of the clip.  Two launches do the same on the device:
//   detect_nms_kernel     one CTA per (clip, class): gathers the centre-frame boxes and the class column straight from
//                         pred_loc / pred_prob (no gather tensors), rank-sorts the candidates above the threshold,
//                         greedy NMS in shared memory (bit-exact predicate above), writes keep / score / normalised box
//                         at candidate index  clip_start * ncls + c * n_clip + j.
//   detect_select_kernel  one CTA per clip: orders the kept candidates as the reference does -- file order (class, tube)
//                         when topk <= 0, else the tuple sort of test.py:205-208, (score, class, j) descending, cut at
//                         topk -- and writes them compactly: det[clip][rank] = {x1, y1, x2, y2, score, class, tube, 0}.
__global__ void __launch_bounds__(128) detect_nms_kernel(const float* __restrict__ prob, int prob_ld,
                                                         const float* __restrict__ loc, int loc_ld,
                                                         const int* __restrict__ clip_offsets, int ncls, float conf,
                                                         float thr, int ge, float vw, float vh, float nw, float nh,
                                                         uint8_t* __restrict__ keep, float* __restrict__ score_out,
                                                         float4* __restrict__ box_out) {
  const int clip = blockIdx.x / ncls, c = blockIdx.x - clip * ncls;
  const int beg = clip_offsets[clip], n = clip_offsets[clip + 1] - beg;
  const size_t cand0 = (size_t)beg * ncls + (size_t)c * n;
  greedy_nms_smem(
      n, thr, ge, [&](int i) { return prob[(size_t)(beg + i) * prob_ld + c]; },
      [&](float s) { return s > conf; },   // test.py:180 scores.gt(conf): false for NaN
      [&](int i, float s) {
        const float4 b = valid_one(ld4(loc + (size_t)(beg + i) * loc_ld), vw, vh);   // test.py:191
        score_out[cand0 + i] = s;
        box_out[cand0 + i] = make_float4(__fdiv_rn(b.x, nw), __fdiv_rn(b.y, nh), __fdiv_rn(b.z, nw), __fdiv_rn(b.w, nh));  // test.py:197-198
        return b;
      },
      [&](int i, uint8_t k) { keep[cand0 + i] = k; });
}

// One CTA per clip.  Pass 1 compacts the kept candidates in candidate order (= the reference's file order: class, tube)
// into shared memory with a ballot scan; pass 2 ranks them (m^2 compares on the m <= kSelMax survivors, all in shared
// memory) when a top-k cut is requested.  Clips with more survivors than kSelMax rank against global memory instead.
constexpr int kSelMax = 4096;
__global__ void __launch_bounds__(256) detect_select_kernel(const uint8_t* __restrict__ keep,
                                                            const float* __restrict__ score, const float4* __restrict__ box,
                                                            const int* __restrict__ clip_offsets, int ncls, int topk,
                                                            int cap, float* __restrict__ det, int* __restrict__ det_count) {
  __shared__ float s_score[kSelMax];
  __shared__ int s_idx[kSelMax];
  const int clip = blockIdx.x;
  const int beg = clip_offsets[clip], n = clip_offsets[clip + 1] - beg;
  const int cands = n * ncls;
  const size_t cand0 = (size_t)beg * ncls;
  // ---- pass 1: kept candidates, ascending candidate index -> slot (prefix count)
  const int m = ballot_compact<8>(cands, [&](int i) { return (int)keep[cand0 + i]; }, [&](int i, int slot) {
    if (slot < kSelMax) { s_idx[slot] = i; s_score[slot] = score[cand0 + i]; }
  });
  const bool in_smem = m <= kSelMax;
  auto emit = [&](int i, float si, int rank) {
    if (rank >= cap) return;
    const float4 b = box[cand0 + i];
    float* o = det + ((size_t)clip * cap + rank) * 8;
    const int c = i / n;
    o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = si; o[5] = (float)c; o[6] = (float)(i - c * n); o[7] = 0.0f;
  };
  if (in_smem) {
    for (int k = threadIdx.x; k < m; k += blockDim.x) {
      const int i = s_idx[k];
      const float si = s_score[k];
      int rank = k;                                   // file order
      if (topk > 0) {
        // (score, class, j) descending (test.py:205-208): inside a class j grows with the tube index and the candidate
        // index is class * n + tube, so "greater (class, j)" == "greater candidate index" == "greater slot"
        rank = 0;
        for (int t = 0; t < m; ++t) {
          const float st = s_score[t];
          rank += (st > si) || (st == si && t > k);
        }
        if (rank >= topk) continue;
      }
      emit(i, si, rank);
    }
  } else {
    for (int i = threadIdx.x; i < cands; i += blockDim.x) {
      if (!keep[cand0 + i]) continue;
      const float si = score[cand0 + i];
      int rank = 0;
      if (topk > 0) {
        for (int t = 0; t < cands; ++t) {
          if (!keep[cand0 + t]) continue;
          const float st = score[cand0 + t];
          rank += (st > si) || (st == si && t > i);
        }
        if (rank >= topk) continue;
      } else {
        for (int t = 0; t < i; ++t) rank += keep[cand0 + t] ? 1 : 0;
      }
      emit(i, si, rank);
    }
  }
  if (threadIdx.x == 0) {
    int k = m;
    if (topk > 0 && k > topk) k = topk;
    det_count[clip] = k < cap ? k : cap;
  }
}

// ---- class-only detections (train_cls.py:505-543): no valid_tubes clamp, no NMS, no top-k --------------------------
// One CTA per clip.  Candidate i = class * n_clip + proposal is the reference's file order (clip, class, proposal
// ascending); the ballot scan thresholds each candidate (scores.gt), counts the passing ones and writes them compactly:
// det[clip][slot] = {x1/nw, y1/nh, x2/nw, y2/nh, score, class, proposal, 0}, box = the proposal's centre frame.
__global__ void __launch_bounds__(256) detect_scores_kernel(const float* __restrict__ prob, int prob_ld,
                                                            const float* __restrict__ box, int box_ld,
                                                            const int* __restrict__ clip_offsets, int ncls, float conf,
                                                            float nw, float nh, int cap, float* __restrict__ det,
                                                            int* __restrict__ det_count) {
  const int clip = blockIdx.x;
  const int beg = clip_offsets[clip], n = clip_offsets[clip + 1] - beg;
  const int cands = n > 0 ? n * ncls : 0;
  auto score = [&](int i) {
    const int c = i / n;
    return prob[(size_t)(beg + i - c * n) * prob_ld + c];
  };
  const int m = ballot_compact<8>(cands, [&](int i) { return (int)(score(i) > conf); }, [&](int i, int slot) {
    if (slot >= cap) return;   // the host sizes cap for every candidate; never write past it
    const int c = i / n, j = i - c * n;
    const float* b = box + (size_t)(beg + j) * box_ld;
    float* o = det + ((size_t)clip * cap + slot) * 8;
    // train_cls.py:533-534, numpy float32 division by the image size
    o[0] = __fdiv_rn(b[0], nw); o[1] = __fdiv_rn(b[1], nh); o[2] = __fdiv_rn(b[2], nw); o[3] = __fdiv_rn(b[3], nh);
    o[4] = score(i); o[5] = (float)c; o[6] = (float)j; o[7] = 0.0f;
  });
  if (threadIdx.x == 0) det_count[clip] = m < cap ? m : cap;
}

// ---- cross-class merge of demo.py:176-198 on step_detect_f32's rows --------------------------------------------------
// Per clip, over the rows in order: a row not yet taken leads a group and takes every later untaken row whose
// compute_box_iou with it is > thresh (float32).  That is greedy NMS with MergePred, so mask_tiles_kernel and
// resolve_kernel find the leaders; their claim hook records which leader took each row (GroupClaim).  Then
// merge_groups_kernel forms the reference's dict: the mean box of each group (np.mean: a sequential float32 sum over the
// members in row order, over float32(count)), one key per distinct mean (bit-equal means are one key: it keeps its first
// group's position and its last group's members) and the rows that results.txt writes, in order.
// Rows of one clip: resolve_kernel keeps a ceil(cap/64)-word row of the bitmask in (default, 48 KB) shared memory.
constexpr int kMergeMaxRows = 48 * 1024 / 8 * kTile;

struct GroupKeep {    // a leader is its own group
  int* group;
  int ld;
  __device__ __forceinline__ void operator()(int z, int i, unsigned k) const {
    if (k) group[(size_t)z * ld + i] = i;
  }
};

struct GroupClaim {
  int* group;
  int ld;
  __device__ __forceinline__ void operator()(int z, int leader, int col_blk, unsigned long long bits) const {
    int* g = group + (size_t)z * ld + col_blk * kTile;
    while (bits) {
      const int b = __ffsll((long long)bits) - 1;
      bits &= bits - 1;
      g[b] = leader;
    }
  }
};

// Exclusive prefix sum in index order over the whole CTA of kWarps warps: calls emit(i, sum of val(t) for t < i) for every
// i in [0, n), and returns the total.
template <int kWarps, class Val, class Emit>
__device__ __forceinline__ int block_scan(int n, Val val, Emit emit) {
  __shared__ int warp_tot[kWarps];
  __shared__ int base_s;
  if (threadIdx.x == 0) base_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int start = 0; start < n; start += blockDim.x) {
    const int i = start + threadIdx.x;
    const int v = (i < n) ? val(i) : 0;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    int off = base_s;
    for (int w = 0; w < wid; ++w) off += warp_tot[w];
    if (i < n) emit(i, off + incl - v);
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < kWarps; ++w) t += warp_tot[w];
      base_s += t;
    }
    __syncthreads();
  }
  return base_s;
}

// Per-clip scratch of merge_groups_kernel, cap entries per clip (ws + clip * cap).
struct MergeScratch {
  int* group;    // [cap] leader of each row (resolve_kernel)
  int* lead;     // [cap] the g-th leader's row
  int* members;  // [cap] members of group g
  int* first;    // [cap] first group with group g's mean
  int* last;     // [cap] last group with group g's mean
  int* key;      // [cap] key index of group g (g its key's first group)
  int* offset;   // [cap] first write-order row of group g's key (g its key's first group)
  float4* mean;  // [cap] mean box of group g
};

__global__ void __launch_bounds__(1024) merge_groups_kernel(const float* __restrict__ det, const int* __restrict__ det_count,
                                                            int cap, MergeScratch ws, float* __restrict__ mbox,
                                                            int* __restrict__ pairs, int* __restrict__ mcount) {
  const int z = blockIdx.x;
  const int n = min(max(det_count[z], 0), cap);
  const size_t o = (size_t)z * cap;
  const int* group = ws.group + o;
  int *lead = ws.lead + o, *members = ws.members + o, *first = ws.first + o, *last = ws.last + o, *key = ws.key + o;
  int* offset = ws.offset + o;
  float* mean = reinterpret_cast<float*>(ws.mean + o);
  const float* rows = det + o * 8;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // 1. the leaders in row order: group g
  const int G = ballot_compact<32>(n, [&](int i) { return (int)(group[i] == i); }, [&](int i, int slot) { lead[slot] = i; });
  // 2. one warp per group: lane c < 4 sums coordinate c over the members in row order, ((0 + b0) + b1) + ..., in float32
  //    (np.add.reduce starts from its identity +0.0, so a sum of -0.0 is +0.0)
  for (int g = wid; g < G; g += nwarps) {
    const int L = lead[g];
    float s = lane < 4 ? __fadd_rn(0.0f, rows[(size_t)L * 8 + lane]) : 0.0f;
    int count = 1;
    for (int base = L + 1; base < n; base += 32) {
      const int i = base + lane;
      unsigned bal = __ballot_sync(0xffffffffu, i < n && group[i] == L);
      count += __popc(bal);
      if (lane < 4)
        while (bal) {
          const int b = __ffs(bal) - 1;
          bal &= bal - 1;
          s = __fadd_rn(s, rows[(size_t)(base + b) * 8 + lane]);
        }
      __syncwarp();
    }
    if (lane < 4) mean[(size_t)g * 4 + lane] = __fdiv_rn(s, (float)count);
    if (lane == 0) members[g] = count;
  }
  __syncthreads();
  // 3. dict keys: groups with bit-equal means share one (str of a float32 round-trips)
  const uint4* mbits = reinterpret_cast<const uint4*>(mean);
  auto same = [](uint4 a, uint4 b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; };
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const uint4 m = mbits[g];
    int f = g, l = g;
    for (int h = 0; h < g; ++h)
      if (same(mbits[h], m)) { f = h; break; }
    for (int h = G - 1; h > g; --h)
      if (same(mbits[h], m)) { l = h; break; }
    first[g] = f;
    last[g] = l;
  }
  __syncthreads();
  // 4. keys in dict order (the first group of each), with their mean box
  const int K = ballot_compact<32>(G, [&](int g) { return (int)(first[g] == g); }, [&](int g, int k) {
    key[g] = k;
    reinterpret_cast<float4*>(mbox)[o + k] = reinterpret_cast<const float4*>(mean)[g];
  });
  // 5. write order: each key's rows are its last group's members
  const int P = block_scan<32>(G, [&](int g) { return first[g] == g ? members[last[g]] : 0; },
                               [&](int g, int off) { offset[g] = off; });
  for (int g = wid; g < G; g += nwarps) {
    if (last[g] != g) continue;   // warp-uniform
    const int L = lead[g], k = key[first[g]];
    int* out = pairs + (o + offset[first[g]]) * 2;
    if (lane == 0) { out[0] = L; out[1] = k; }
    int r = 1;
    for (int base = L + 1; base < n; base += 32) {
      const int i = base + lane;
      const bool mine = i < n && group[i] == L;
      const unsigned bal = __ballot_sync(0xffffffffu, mine);
      if (mine) {
        const int at = r + __popc(bal & ((1u << lane) - 1));
        out[at * 2] = i;
        out[at * 2 + 1] = k;
      }
      r += __popc(bal);
    }
  }
  if (threadIdx.x == 0) { mcount[z * 2] = K; mcount[z * 2 + 1] = P; }
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace step

using namespace step;

extern "C" size_t step_nms_workspace_bytes(int n) {
  if (n <= 0) return 256;
  size_t cb = (size_t)ceil_div(n, kTile);
  return align256((size_t)n * sizeof(float4)) + align256((size_t)n * sizeof(int)) +
         align256((size_t)n * cb * sizeof(unsigned long long)) + align256((size_t)n) + 256;
}

extern "C" int step_nms_f32(const float* boxes, const float* scores, int n, float thr, int ge,
                            int64_t* keep_out, int* n_keep, void* workspace, size_t ws_bytes,
                            step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0 && n_keep != nullptr, "step_nms_f32: bad n / n_keep");
  cudaStream_t s = cu(stream);
  if (n == 0) {  // nms_cpu.cpp:37-39: empty in, empty out
    cudaError_t e = cudaMemsetAsync(n_keep, 0, sizeof(int), s);
    return e == cudaSuccess ? 0 : fail((int)e, "step_nms_f32: memset: %s", cudaGetErrorString(e));
  }
  STEP_CHECK_ARG(boxes && scores && keep_out && workspace, "step_nms_f32: null pointer");
  STEP_CHECK_ARG(((uintptr_t)boxes & 15) == 0, "step_nms_f32: boxes must be 16-byte aligned");
  const int cb = ceil_div(n, kTile);
  STEP_CHECK_ARG((size_t)cb * 8 <= 200 * 1024, "step_nms_f32: n too large (max %d)", 200 * 1024 / 8 * kTile);
  if (ws_bytes < step_nms_workspace_bytes(n))
    return fail(STEP_E_WORKSPACE, "step_nms_f32: workspace %zu < %zu", ws_bytes, step_nms_workspace_bytes(n));
  char* w = (char*)workspace;
  float4* sorted = (float4*)w;  w += align256((size_t)n * sizeof(float4));
  int* order = (int*)w;         w += align256((size_t)n * sizeof(int));
  unsigned long long* mask = (unsigned long long*)w;  w += align256((size_t)n * cb * sizeof(unsigned long long));
  uint8_t* flag = (uint8_t*)w;

  nms_rank_kernel<<<ceil_div(n, 256), 256, 0, s>>>(boxes, scores, n, sorted, order);
  STEP_LAUNCH_CHECK("nms_rank_kernel");
  const SortedRows rows{sorted, n};
  mask_tiles_kernel<<<dim3(cb, cb), kTile, 0, s>>>(rows, NmsPred{thr, ge}, cb, 0, mask);
  STEP_LAUNCH_CHECK("mask_tiles_kernel");
  size_t smem = (size_t)cb * sizeof(unsigned long long);
  auto resolve = resolve_kernel<SortedRows, KeepByOrder, NoClaim>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(resolve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "step_nms_f32: smem attr: %s", cudaGetErrorString(e));
  }
  resolve<<<1, 1024, smem, s>>>(mask, rows, cb, 0, KeepByOrder{order, flag}, NoClaim{});
  STEP_LAUNCH_CHECK("resolve_kernel");
  nms_compact_kernel<<<1, 1024, 0, s>>>(flag, n, keep_out, n_keep);
  STEP_LAUNCH_CHECK("nms_compact_kernel");
  return 0;
}

extern "C" int step_nms_segmented_f32(const float* boxes, const float* scores, const int* seg_offsets,
                                      int n_seg, float thr, int ge, float min_score, uint8_t* keep_mask,
                                      step_stream_t stream) {
  STEP_CHECK_ARG(n_seg >= 0, "step_nms_segmented_f32: n_seg < 0");
  if (n_seg == 0) return 0;
  STEP_CHECK_ARG(boxes && scores && seg_offsets && keep_mask, "step_nms_segmented_f32: null pointer");
  STEP_CHECK_ARG(((uintptr_t)boxes & 15) == 0, "step_nms_segmented_f32: boxes must be 16-byte aligned");
  nms_segmented_kernel<<<n_seg, 256, 0, cu(stream)>>>(boxes, scores, seg_offsets, thr, ge, min_score, keep_mask);
  STEP_LAUNCH_CHECK("nms_segmented_kernel");
  return 0;
}

extern "C" int step_nms_segmented_max_rows(void) { return kSegMax; }

extern "C" int step_detect_f32(const float* prob, int prob_ld, const float* loc, int loc_ld, const int* clip_offsets,
                               int n_clips, int n_rows, int max_per_clip, int ncls, float conf_thresh, float nms_thresh,
                               int ge, float valid_w, float valid_h, float norm_w, float norm_h, int topk, int cap,
                               uint8_t* keep, float* score, float* box, float* det, int* det_count,
                               step_stream_t stream) {
  STEP_CHECK_ARG(n_clips >= 0 && n_rows >= 0 && ncls > 0, "step_detect_f32: bad sizes");
  if (n_clips == 0) return 0;
  STEP_CHECK_ARG(max_per_clip <= kSegMax, "step_detect_f32: %d tubes in one clip (max %d per (clip, class) problem)",
                 max_per_clip, kSegMax);
  STEP_CHECK_ARG(prob && loc && clip_offsets && keep && score && box && det && det_count, "step_detect_f32: null pointer");
  STEP_CHECK_ARG(prob_ld >= ncls && loc_ld >= 4 && cap > 0, "step_detect_f32: bad strides / cap");
  STEP_CHECK_ARG(((uintptr_t)box & 15) == 0, "step_detect_f32: box must be 16-byte aligned");
  cudaStream_t s = cu(stream);
  detect_nms_kernel<<<n_clips * ncls, 128, 0, s>>>(prob, prob_ld, loc, loc_ld, clip_offsets, ncls, conf_thresh, nms_thresh,
                                                   ge, valid_w, valid_h, norm_w, norm_h, keep, score, (float4*)box);
  STEP_LAUNCH_CHECK("detect_nms_kernel");
  detect_select_kernel<<<n_clips, 256, 0, s>>>(keep, score, (const float4*)box, clip_offsets, ncls, topk, cap, det, det_count);
  STEP_LAUNCH_CHECK("detect_select_kernel");
  return 0;
}

extern "C" int step_detect_scores_check(const float* prob, int prob_ld, const float* box, int box_ld, const int* clip_offsets,
                                        int n_clips, int n_rows, int max_per_clip, int ncls, int cap, const float* det,
                                        const int* det_count) {
  STEP_CHECK_ARG(n_clips >= 0 && n_rows >= 0 && ncls > 0 && max_per_clip >= 0 && max_per_clip <= n_rows,
                 "step_detect_scores_f32: bad sizes (n_clips %d, n_rows %d, max_per_clip %d, ncls %d)", n_clips, n_rows,
                 max_per_clip, ncls);
  if (n_clips == 0) return 0;
  STEP_CHECK_ARG(prob && box && clip_offsets && det && det_count, "step_detect_scores_f32: null pointer");
  STEP_CHECK_ARG(prob_ld >= ncls && box_ld >= 4, "step_detect_scores_f32: bad strides (prob_ld %d, box_ld %d)", prob_ld, box_ld);
  STEP_CHECK_ARG(cap > 0 && (long long)max_per_clip * ncls <= cap,
                 "step_detect_scores_f32: cap %d below max_per_clip %d * ncls %d", cap, max_per_clip, ncls);
  return 0;
}

extern "C" int step_detect_scores_f32(const float* prob, int prob_ld, const float* box, int box_ld, const int* clip_offsets,
                                      int n_clips, int n_rows, int max_per_clip, int ncls, float conf_thresh, float norm_w,
                                      float norm_h, int cap, float* det, int* det_count, step_stream_t stream) {
  const int rc = step_detect_scores_check(prob, prob_ld, box, box_ld, clip_offsets, n_clips, n_rows, max_per_clip, ncls, cap,
                                          det, det_count);
  if (rc || n_clips == 0) return rc;
  detect_scores_kernel<<<n_clips, 256, 0, cu(stream)>>>(prob, prob_ld, box, box_ld, clip_offsets, ncls, conf_thresh, norm_w,
                                                        norm_h, cap, det, det_count);
  STEP_LAUNCH_CHECK("detect_scores_kernel");
  return 0;
}

// Workspace of step_detect_merge_f32, per clip: the bitmask (cap rows of ceil(cap/64) words), then MergeScratch.
static size_t merge_mask_bytes(int cap) { return align256((size_t)cap * ceil_div(cap, kTile) * sizeof(unsigned long long)); }
static size_t merge_ints_bytes(int n_clips, int cap) { return align256((size_t)n_clips * cap * sizeof(int)); }

extern "C" size_t step_detect_merge_workspace_bytes(int n_clips, int cap) {
  if (n_clips <= 0 || cap <= 0) return 256;
  return (size_t)n_clips * merge_mask_bytes(cap) + 7 * merge_ints_bytes(n_clips, cap) +
         align256((size_t)n_clips * cap * sizeof(float4)) + 256;
}

extern "C" int step_detect_merge_max_rows(void) { return kMergeMaxRows; }

extern "C" int step_detect_merge_f32(const float* det, const int* det_count, int n_clips, int cap, float thresh, float* mbox,
                                     int* pairs, int* mcount, void* workspace, size_t ws_bytes, step_stream_t stream) {
  STEP_CHECK_ARG(n_clips >= 0 && n_clips <= 65535, "step_detect_merge_f32: n_clips %d (0..65535)", n_clips);
  STEP_CHECK_ARG(cap > 0 && cap <= kMergeMaxRows, "step_detect_merge_f32: cap %d (1..%d)", cap, kMergeMaxRows);
  if (n_clips == 0) return 0;
  STEP_CHECK_ARG(det && det_count && mbox && pairs && mcount && workspace, "step_detect_merge_f32: null pointer");
  STEP_CHECK_ARG(((uintptr_t)det & 15) == 0 && ((uintptr_t)mbox & 15) == 0 && ((uintptr_t)workspace & 255) == 0,
                 "step_detect_merge_f32: det / mbox must be 16-byte and the workspace 256-byte aligned");
  const size_t need = step_detect_merge_workspace_bytes(n_clips, cap);
  STEP_CHECK_ARG(ws_bytes >= need, "step_detect_merge_f32: workspace %zu < %zu bytes", ws_bytes, need);
  char* w = (char*)workspace;
  unsigned long long* mask = (unsigned long long*)w;
  w += (size_t)n_clips * merge_mask_bytes(cap);
  MergeScratch ms;
  int** ints[7] = {&ms.group, &ms.lead, &ms.members, &ms.first, &ms.last, &ms.key, &ms.offset};
  for (int k = 0; k < 7; ++k) { *ints[k] = (int*)w; w += merge_ints_bytes(n_clips, cap); }
  ms.mean = (float4*)w;
  const int cb = ceil_div(cap, kTile);
  const size_t stride = merge_mask_bytes(cap) / sizeof(unsigned long long);
  const DetRows rows{det, det_count, cap};
  cudaStream_t s = cu(stream);
  mask_tiles_kernel<<<dim3(cb, cb, n_clips), kTile, 0, s>>>(rows, MergePred{thresh}, cb, stride, mask);
  STEP_LAUNCH_CHECK("mask_tiles_kernel");
  resolve_kernel<<<n_clips, 1024, (size_t)cb * sizeof(unsigned long long), s>>>(mask, rows, cb, stride, GroupKeep{ms.group, cap},
                                                                               GroupClaim{ms.group, cap});
  STEP_LAUNCH_CHECK("resolve_kernel");
  merge_groups_kernel<<<n_clips, 1024, 0, s>>>(det, det_count, cap, ms, mbox, pairs, mcount);
  STEP_LAUNCH_CHECK("merge_groups_kernel");
  return 0;
}
