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

__device__ __forceinline__ bool suppresses(float4 a, float area_a, float4 b, float area_b, float thr, int ge) {
  // nms_cpu.cpp:74-85
  float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
  float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
  float w = fmaxf(0.0f, __fadd_rn(__fsub_rn(xx2, xx1), 1.0f));
  float h = fmaxf(0.0f, __fadd_rn(__fsub_rn(yy2, yy1), 1.0f));
  float inter = __fmul_rn(w, h);
  float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
  return ge ? (ovr >= thr) : (ovr > thr);
}

// ---- 1. ordering: rank sort (score desc, index asc).  O(n^2) compares, embarrassingly parallel;
//         10k boxes = 1e8 compares ~ 10 us.  Deterministic and stable by construction, unlike the
//         reference's torch.sort (unstable for n > 16).
__global__ void __launch_bounds__(256) nms_rank_kernel(const float* __restrict__ boxes,
                                                       const float* __restrict__ scores, int n,
                                                       float4* __restrict__ sorted_boxes,
                                                       int* __restrict__ order) {
  __shared__ float tile[1024];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  float si = i < n ? scores[i] : 0.0f;
  int rank = 0;
  for (int base = 0; base < n; base += 1024) {
    int cnt = min(1024, n - base);
    for (int t = threadIdx.x; t < cnt; t += blockDim.x) tile[t] = scores[base + t];
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

// ---- 2. upper-triangular 64x64 bitmask tiles on the sorted boxes
constexpr int kTile = 64;
__global__ void __launch_bounds__(kTile) nms_mask_kernel(const float4* __restrict__ sb, int n, float thr,
                                                         int ge, int col_blocks,
                                                         unsigned long long* __restrict__ mask) {
  const int row_blk = blockIdx.y, col_blk = blockIdx.x;
  if (col_blk < row_blk) return;  // never read by the resolve
  __shared__ float4 cb[kTile];
  __shared__ float ca[kTile];
  const int col_size = min(n - col_blk * kTile, kTile);
  if (threadIdx.x < col_size) {
    float4 b = sb[col_blk * kTile + threadIdx.x];
    cb[threadIdx.x] = b;
    ca[threadIdx.x] = box_area(b);
  }
  __syncthreads();
  const int r = row_blk * kTile + threadIdx.x;
  if (r < n) {
    float4 a = sb[r];
    float aa = box_area(a);
    unsigned long long bits = 0;
    int start = (row_blk == col_blk) ? threadIdx.x + 1 : 0;
    for (int j = start; j < col_size; ++j)
      if (suppresses(a, aa, cb[j], ca[j], thr, ge)) bits |= 1ULL << j;
    mask[(size_t)r * col_blocks + col_blk] = bits;
  }
}

// ---- 3. greedy resolve on device: one CTA walks the 64-box blocks in score order.
__global__ void __launch_bounds__(1024) nms_resolve_kernel(const unsigned long long* __restrict__ mask,
                                                           const int* __restrict__ order, int n,
                                                           int col_blocks, uint8_t* __restrict__ keep_flag) {
  extern __shared__ unsigned long long remv[];  // [col_blocks]
  __shared__ unsigned long long diag[kTile];
  __shared__ unsigned long long kept_s;
  for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) remv[j] = 0;
  __syncthreads();
  for (int blk = 0; blk < col_blocks; ++blk) {
    const int cnt = min(kTile, n - blk * kTile);
    if (threadIdx.x < cnt) diag[threadIdx.x] = mask[(size_t)(blk * kTile + threadIdx.x) * col_blocks + blk];
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long r = remv[blk], kept = 0;
      for (int b = 0; b < cnt; ++b)
        if (!((r >> b) & 1ULL)) { kept |= 1ULL << b; r |= diag[b]; }
      kept_s = kept;
    }
    __syncthreads();
    const unsigned long long kept = kept_s;
    if (threadIdx.x < cnt) keep_flag[order[blk * kTile + threadIdx.x]] = (uint8_t)((kept >> threadIdx.x) & 1ULL);
    for (int j = blk + 1 + threadIdx.x; j < col_blocks; j += blockDim.x) {
      unsigned long long acc = remv[j], k = kept;
      while (k) {
        int b = __ffsll((long long)k) - 1;
        k &= k - 1;
        acc |= mask[(size_t)(blk * kTile + b) * col_blocks + j];
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
//      are dropped.  The caller says how rows are read and where their keep flags go:
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
      [&](float s) { return s >= min_score; },   // the confidence threshold of test.py:183
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
      [&](float s) { return s > conf; },   // test.py:183 scores.gt(conf)
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
  nms_mask_kernel<<<dim3(cb, cb), kTile, 0, s>>>(sorted, n, thr, ge, cb, mask);
  STEP_LAUNCH_CHECK("nms_mask_kernel");
  size_t smem = (size_t)cb * sizeof(unsigned long long);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(nms_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "step_nms_f32: smem attr: %s", cudaGetErrorString(e));
  }
  nms_resolve_kernel<<<1, 1024, smem, s>>>(mask, order, n, cb, flag);
  STEP_LAUNCH_CHECK("nms_resolve_kernel");
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
