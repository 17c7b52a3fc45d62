// train.cu -- the first pieces of the training step (SURVEY.md section 8f rank 1; train.py:286-348 of the reference):
//   * head_losses_kernel       TwoBranchNet's three losses (models/two_branch.py:276-333) and, in the same pass, the
//                              gradient of the training objective  mean(loss_cls) + w_loc * loss_loc + w_nb * loss_nb
//                              (train.py:323-347) with respect to the head outputs;
//   * cls_loss_kernel          the loss of class-only heads (TwoBranchNet(cls_only=True), the first training stage of
//                              train_cls.py) and d mean(loss_cls) / d logits, with the classification arithmetic of
//                              head_losses_kernel (one shared device function);
//   * roi_align_bwd_nhwc       channels-last ROIAlign backward WITHOUT float atomics: every feature pixel gathers its
//                              contributions in a fixed order (ROI index, bin, sample), so the result is bit-for-bit
//                              repeatable -- the reference's RoIAlignBackwardFeature (cuda/ROIAlign_cuda.cu:201-278) scatters
//                              with atomicAdd and is not;
//   * roi_align_bwd_slice_nhwc the same backward for ROIs pooled from a temporal slice of conv_feat (temporal mode of
//                              train.py:294-309), accumulated into the gradient of the whole feature map;
//   * ctx_grad_reduce          the gradient of ContextNet's output from the per-tube context inputs of the classifier
//                              (train.py:317-321), summed per clip in tube order and spread over the step's frames;
//   * linear_bwd_*             backward of the small-N linears of the head (global_cls, local_reg, neighbor_reg*):
//                              dx = dy W, dW = dy^T x, db = sum dy, fixed summation order;
//   * conv1x1_wgrad_*          weight gradient of a 1x1(x1) convolution, dW[Cout, Cin] = dz^T x with the reduction over
//                              the pixels on the tensor cores (fp16 operands, fp32 accumulate), split over pixel chunks with
//                              a fixed-order second pass.
// All fp32 arithmetic of the losses is explicitly rounded in the reference's operand order; exp / log are the only
// operations that are not bit-exact (tolerance stated in tests/test_gpu_train.py).
#include <math.h>

#include <algorithm>

#include <mma.h>

#include "common.cuh"
#include "dropout.cuh"
#include "roi_math.cuh"
#include "tube_math.cuh"

namespace step {

// ---- losses -------------------------------------------------------------------------------------------------------
// F.smooth_l1_loss(beta = 1): 0.5 d^2 if |d| < 1 else |d| - 0.5; derivative d | sign(d)
__device__ __forceinline__ float smooth_l1(float d, float* grad) {
  const float ad = fabsf(d);
  if (ad < 1.0f) { *grad = d; return __fmul_rn(__fmul_rn(0.5f, d), d); }
  *grad = d > 0.0f ? 1.0f : -1.0f;
  return __fsub_rn(ad, 0.5f);
}

// Sum of the centre rows' classification masks, targets[n][1][4], in tube order (two_branch.py:291-293).  One thread.
__device__ __forceinline__ float cls_mask_sum(const float* __restrict__ targets, int N, int tgt_ld) {
  float mc = 0.0f;
  for (int n = 0; n < N; ++n) mc = __fadd_rn(mc, targets[((size_t)n * 3 + 1) * tgt_ld + 4]);
  return mc;
}

// Classification loss of the centre chunk (two_branch.py:291-297) over the [N, cls] logits, block-strided: BCE with logits
// against the labels masked by the centre row's classification flag, and d mean(loss_cls) / d logit.  Without any
// classification sample (has_cls false) both are zero.  Shared by head_losses_kernel and cls_loss_kernel so that the two
// agree bit for bit.
__device__ __forceinline__ void cls_loss_pass(const float* __restrict__ logits, const float* __restrict__ targets, int N, int cls,
                                              int tgt_ld, bool has_cls, float* __restrict__ loss_cls, float* __restrict__ dlogits) {
  const float inv_ncls = 1.0f / (float)((long long)N * cls);
  for (int i = threadIdx.x; i < N * cls; i += blockDim.x) {
    const int n = i / cls, c = i - n * cls;
    const float x = logits[i];
    float l = 0.0f, gx = 0.0f;
    if (has_cls) {
      const float* tc = targets + ((size_t)n * 3 + 1) * tgt_ld;
      const float t = __fmul_rn(tc[6 + c], tc[4]);
      // ATen: (1 - t) * x - log_sigmoid(x),  log_sigmoid(x) = min(x, 0) - log1p(exp(-|x|))
      const float ls = __fsub_rn(fminf(x, 0.0f), log1pf(expf(-fabsf(x))));
      l = __fsub_rn(__fmul_rn(__fsub_rn(1.0f, t), x), ls);
      const float sg = 1.0f / (1.0f + expf(-x));
      gx = __fmul_rn(__fsub_rn(sg, t), inv_ncls);              // d mean(loss_cls) / d logit
    }
    loss_cls[i] = l;
    if (dlogits) dlogits[i] = gx;
  }
}

struct LossGeom {
  int N, cls, T_len, Tc;     // tubes, classes, frames of local_loc, frames of first/last_loc (= T)
  int centre, first_idx, last_idx, half_T;   // chunk_idx[chunks/2], chunk_idx[0], chunk_idx[-1] (two_branch.py:226-228)
  int s0, e0;                // first / last chunk start inside local_loc (two_branch.py:265-266)
  int tgt_ld;                // 6 + cls
  float w_loc, w_nb;         // lambda_reg, lambda_neighbor (train.py:335-336)
};

// One CTA.  Sums are taken in tube order by one thread after a block-wide staging pass: N is a few hundred at most and
// this keeps the reductions bit-for-bit repeatable.
__global__ void __launch_bounds__(256) head_losses_kernel(LossGeom g, const float* __restrict__ logits,
                                                          const float* __restrict__ local_loc, const float* __restrict__ first_loc,
                                                          const float* __restrict__ last_loc, const float* __restrict__ tubes,
                                                          const float* __restrict__ targets, float* __restrict__ loss_cls,
                                                          float* __restrict__ loss_loc, float* __restrict__ loss_nb,
                                                          int* __restrict__ flags, float* __restrict__ dlogits,
                                                          float* __restrict__ dloc, float* __restrict__ dfirst,
                                                          float* __restrict__ dlast, float* __restrict__ scratch) {
  __shared__ float s_sum[3];   // sum of cls mask, loc mask x4, neighbour mask x4
  __shared__ float s_loss[2];
  const int N = g.N;
  // targets[n][j] with j = 0 first, 1 centre, 2 last (two_branch.py:283-285: [:, 0], [:, 1], [:, -1])
  auto tgt = [&](int n, int j) { return targets + ((size_t)n * 3 + j) * g.tgt_ld; };
  if (threadIdx.x == 0) {
    const float mc = cls_mask_sum(targets, N, g.tgt_ld);
    float ml = 0.0f, mn = 0.0f;
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) ml = __fadd_rn(ml, tgt(n, 1)[5]);
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) mn = __fadd_rn(mn, tgt(n, 0)[5]);
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) mn = __fadd_rn(mn, tgt(n, 2)[5]);
    s_sum[0] = mc; s_sum[1] = ml; s_sum[2] = mn;
    flags[0] = mc != 0.0f; flags[1] = ml != 0.0f; flags[2] = mn != 0.0f;
  }
  __syncthreads();
  const bool has_cls = s_sum[0] != 0.0f, has_loc = s_sum[1] != 0.0f, has_nb = s_sum[2] != 0.0f;
  // ---- classification: BCE with logits on the centre chunk, background samples masked (two_branch.py:291-297)
  cls_loss_pass(logits, targets, N, g.cls, g.tgt_ld, has_cls, loss_cls, dlogits);
  // ---- regression: per-tube smooth-L1 terms staged in `scratch` [N][3][4] (loss) and gradients written in place
  if (dloc) for (int i = threadIdx.x; i < N * g.T_len * 4; i += blockDim.x) dloc[i] = 0.0f;
  if (dfirst) for (int i = threadIdx.x; i < N * g.Tc * 4; i += blockDim.x) { dfirst[i] = 0.0f; dlast[i] = 0.0f; }
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    const float* tb = tubes + (size_t)n * g.T_len * 5;
    float enc[4], gr;
    // centre (two_branch.py:301-311)
    st4(enc, encode_one(ld4(tgt(n, 1)), ld4(tb + (size_t)g.centre * 5 + 1)));
    const float mloc = tgt(n, 1)[5];
    for (int k = 0; k < 4; ++k) {
      const float d = __fsub_rn(local_loc[((size_t)n * g.T_len + g.centre) * 4 + k], enc[k]);
      const float l = smooth_l1(d, &gr);
      scratch[((size_t)n * 3 + 0) * 4 + k] = __fmul_rn(l, mloc);
      if (dloc && has_loc) dloc[((size_t)n * g.T_len + g.centre) * 4 + k] = __fdiv_rn(__fmul_rn(__fmul_rn(gr, mloc), g.w_loc), s_sum[1]);
    }
    // neighbours (two_branch.py:315-333): first then last
    for (int j = 0; j < 2; ++j) {
      const int tj = j == 0 ? 0 : 2, idx = j == 0 ? g.first_idx : g.last_idx;
      const float* pred = (j == 0 ? first_loc : last_loc) + ((size_t)n * g.Tc + g.half_T) * 4;
      float* dpred = (j == 0 ? dfirst : dlast);
      st4(enc, encode_one(ld4(tgt(n, tj)), ld4(tb + (size_t)idx * 5 + 1)));
      const float m = tgt(n, tj)[5];
      for (int k = 0; k < 4; ++k) {
        const float d = __fsub_rn(pred[k], enc[k]);
        const float l = smooth_l1(d, &gr);
        scratch[((size_t)n * 3 + 1 + j) * 4 + k] = __fmul_rn(l, m);
        if (dpred && has_nb) dpred[((size_t)n * g.Tc + g.half_T) * 4 + k] = __fdiv_rn(__fmul_rn(__fmul_rn(gr, m), g.w_nb), s_sum[2]);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sl = 0.0f, sn = 0.0f;
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) sl = __fadd_rn(sl, scratch[((size_t)n * 3 + 0) * 4 + k]);
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) sn = __fadd_rn(sn, scratch[((size_t)n * 3 + 1) * 4 + k]);   // cat([first, last])
    for (int n = 0; n < N; ++n) for (int k = 0; k < 4; ++k) sn = __fadd_rn(sn, scratch[((size_t)n * 3 + 2) * 4 + k]);
    s_loss[0] = has_loc ? __fdiv_rn(sl, s_sum[1]) : 0.0f;
    s_loss[1] = has_nb ? __fdiv_rn(sn, s_sum[2]) : 0.0f;
    loss_loc[0] = s_loss[0];
    loss_nb[0] = s_loss[1];
  }
  __syncthreads();
  // first_loc / last_loc are slices of local_loc plus the neighbour regressors (two_branch.py:265-270): their gradient
  // also flows into local_loc at the slice positions
  if (dloc && dfirst) {
    for (int i = threadIdx.x; i < N * g.Tc * 4; i += blockDim.x) {
      const int n = i / (g.Tc * 4), r = i - n * g.Tc * 4;
      const float a = dfirst[i], b = dlast[i];
      // element (n, r) belongs to this thread alone: the [s0, s0 + Tc) and [e0, e0 + Tc) ranges are either identical
      // (one chunk) or disjoint, so the two updates never race and their order is fixed
      if (a != 0.0f) dloc[((size_t)n * g.T_len + g.s0) * 4 + r] += a;
      if (b != 0.0f) dloc[((size_t)n * g.T_len + g.e0) * 4 + r] += b;
    }
  }
}

// The loss of class-only heads (TwoBranchNet(cls_only=True), two_branch.py:291-297): the classification part of
// head_losses_kernel alone, with no regression inputs.  One CTA.
__global__ void __launch_bounds__(256) cls_loss_kernel(int N, int cls, const float* __restrict__ logits,
                                                       const float* __restrict__ targets, float* __restrict__ loss_cls,
                                                       int* __restrict__ flags, float* __restrict__ dlogits) {
  __shared__ float s_mc;
  if (threadIdx.x == 0) {
    s_mc = cls_mask_sum(targets, N, 6 + cls);
    flags[0] = s_mc != 0.0f;
  }
  __syncthreads();
  cls_loss_pass(logits, targets, N, cls, 6 + cls, s_mc != 0.0f, loss_cls, dlogits);
}

// ---- ROIAlign backward, channels-last, deterministic ----------------------------------------------------------------
// grad_in[k][h][w][c] = sum over ROIs r on frame k (ascending r), bins (ph, pw) and samples (iy, ix) in loop order of
//   w_tap(r, bin, sample, this pixel) * grad_out[r][bin][c] / count(r)        (ROIAlign_cuda.cu:201-278)
// One CTA per (frame, pixel row); the per-ROI sample table (each sample's Tap and bin, sampled exactly as the forward in
// roi.cu) is built in shared memory by the CTA and scanned by every (pixel, channel vector) thread.  No atomics: a thread
// owns its output element.
struct RoiBwdSample { Tap tap; int bin; };

// Adds the contributions of every ROI r with roi[0] == roi_frame to dst, this frame's [H*W, C] gradient (channel stride
// dst_ld), which the caller has initialised: per ROI and element the samples are summed in a fixed order and the sum is
// added to dst.  Called by the whole CTA; `tab` is the CTA's shared sample table.
template <typename T>
__device__ __forceinline__ void roi_align_bwd_frame(const T* __restrict__ grad_out, int out_ld, const float* __restrict__ rois,
                                                    int R, float scale, int H, int W, int C, int ph, int pw, int sampling_ratio,
                                                    int roi_frame, float* __restrict__ dst, int dst_ld, RoiBwdSample* tab) {
  constexpr int VN = 4;
  const int nvec = C / VN, npix = H * W;
  for (int r = 0; r < R; ++r) {
    const float* roi = rois + 5 * (size_t)r;
    if ((int)roi[0] != roi_frame) continue;                   // uniform across the CTA
    const RoiGeom g = roi_geometry(roi, scale, ph, pw, sampling_ratio);
    const int per_bin = g.gh * g.gw, total = ph * pw * per_bin;
    for (int base = 0; base < total; base += kMaxTaps) {
      const int cnt = min(kMaxTaps, total - base);
      __syncthreads();                                        // the previous table has been consumed
      for (int s = threadIdx.x; s < cnt; s += blockDim.x) {
        const int gidx = base + s;
        const int bin = gidx / per_bin, rem = gidx - bin * per_bin;
        const int iy = rem / g.gw, ix = rem - iy * g.gw;
        const int p = bin / pw, q = bin - p * pw;
        const float y = sample_coord(g.start_h, p, g.bin_h, iy, g.gh), x = sample_coord(g.start_w, q, g.bin_w, ix, g.gw);
        tab[s] = RoiBwdSample{make_tap(H, W, y, x), bin};
      }
      __syncthreads();
      const T* go = grad_out + (size_t)r * ph * pw * out_ld;
      for (int i = threadIdx.x; i < npix * nvec; i += blockDim.x) {
        const int p = i / nvec, cv = i - p * nvec;
        float acc[VN] = {0.f, 0.f, 0.f, 0.f};
        bool hit = false;
        for (int s = 0; s < cnt; ++s) {
          const RoiBwdSample& e = tab[s];
          // the four taps in order; ROIAlign_cuda.cu:263-271: g = top_diff * w / count
          auto add_tap = [&](int pix, float w) {
            if (pix != p) return;
            float gv[VN];
            if constexpr (sizeof(T) == 4) {
              const float4 v = *reinterpret_cast<const float4*>(go + (size_t)e.bin * out_ld + cv * VN);
              gv[0] = v.x; gv[1] = v.y; gv[2] = v.z; gv[3] = v.w;
            } else {
              const uint2 raw = *reinterpret_cast<const uint2*>(go + (size_t)e.bin * out_ld + cv * VN);
              const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
              const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
              gv[0] = a.x; gv[1] = a.y; gv[2] = b.x; gv[3] = b.y;
            }
#pragma unroll
            for (int c = 0; c < VN; ++c) acc[c] = __fadd_rn(acc[c], __fdiv_rn(__fmul_rn(gv[c], w), g.count));
            hit = true;
          };
          add_tap(e.tap.p1, e.tap.w1);
          add_tap(e.tap.p2, e.tap.w2);
          add_tap(e.tap.p3, e.tap.w3);
          add_tap(e.tap.p4, e.tap.w4);
        }
        if (hit) {
          float4* d = reinterpret_cast<float4*>(dst + (size_t)p * dst_ld + cv * VN);
          float4 cur = *d;
          cur.x = __fadd_rn(cur.x, acc[0]); cur.y = __fadd_rn(cur.y, acc[1]); cur.z = __fadd_rn(cur.z, acc[2]); cur.w = __fadd_rn(cur.w, acc[3]);
          *d = cur;
        }
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) roi_align_bwd_nhwc_kernel(const T* __restrict__ grad_out, int out_ld,
                                                                 const float* __restrict__ rois, int R, float scale, int H,
                                                                 int W, int C, int ph, int pw, int sampling_ratio,
                                                                 float* __restrict__ grad_in, int in_ld) {
  __shared__ RoiBwdSample tab[kMaxTaps];
  const int frame = blockIdx.x;
  const int nvec = C / 4, npix = H * W;
  float* dst = grad_in + (size_t)frame * npix * in_ld;
  // this CTA owns grad_in[frame]: zero it, then accumulate ROI by ROI (ascending index: fixed order)
  for (int i = threadIdx.x; i < npix * nvec; i += blockDim.x) {
    const int p = i / nvec, cv = i - p * nvec;
    *reinterpret_cast<float4*>(dst + (size_t)p * in_ld + cv * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  roi_align_bwd_frame<T>(grad_out, out_ld, rois, R, scale, H, W, C, ph, pw, sampling_ratio, frame, dst, in_ld, tab);
}

// The same backward for ROIs whose frame index f is relative to the slice conv_feat[:, t_start:t_start+roi_T]
// (ROINet.pool_into's frame map): one CTA per ROI frame f forms the frame's whole contribution in its [H*W, C] workspace
// frame exactly as roi_align_bwd_nhwc_kernel does, then adds it to grad_in frame (f / roi_T) * feat_T + t_start + f % roi_T.
// Frames outside the slice are not touched, so successive refinement steps accumulate into one [B*feat_T, H, W, C] buffer.
template <typename T>
__global__ void __launch_bounds__(256) roi_align_bwd_slice_nhwc_kernel(const T* __restrict__ grad_out, int out_ld,
                                                                       const float* __restrict__ rois, int R, float scale, int H,
                                                                       int W, int C, int ph, int pw, int sampling_ratio, int roi_T,
                                                                       int feat_T, int t_start, float* __restrict__ ws,
                                                                       float* __restrict__ grad_in, int in_ld) {
  __shared__ RoiBwdSample tab[kMaxTaps];
  const int f = blockIdx.x;
  const int nvec = C / 4, npix = H * W;
  float* part = ws + (size_t)f * npix * C;
  for (int i = threadIdx.x; i < npix * nvec; i += blockDim.x)
    *reinterpret_cast<float4*>(part + (size_t)i * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
  roi_align_bwd_frame<T>(grad_out, out_ld, rois, R, scale, H, W, C, ph, pw, sampling_ratio, f, part, C, tab);
  __syncthreads();
  float* dst = grad_in + ((size_t)(f / roi_T) * feat_T + t_start + f % roi_T) * npix * in_ld;
  for (int i = threadIdx.x; i < npix * nvec; i += blockDim.x) {
    const int p = i / nvec, cv = i - p * nvec;
    const float4 a = *reinterpret_cast<const float4*>(part + (size_t)i * 4);
    float4* d = reinterpret_cast<float4*>(dst + (size_t)p * in_ld + cv * 4);
    float4 cur = *d;
    cur.x = __fadd_rn(cur.x, a.x); cur.y = __fadd_rn(cur.y, a.y); cur.z = __fadd_rn(cur.z, a.z); cur.w = __fadd_rn(cur.w, a.w);
    *d = cur;
  }
}

// ---- ROIPool backward on a frame slice (the reference's ROIPool_cuda.cu:103-132 scatters with atomicAdd) -----------------
// One CTA per (ROI frame f, chunk of `blockDim.x` channels) holds the frame's [H*W, chunk] fp32 accumulator in shared
// memory; thread t owns channel c0 + t (and, at 32 channels or more, shared-memory bank t % 32).  The CTA streams the ROI rows in ascending order,
// compacts those of frame f (in order, blockDim.x rows at a time: no cap on R, no workspace), and every thread adds
// grad_out[row, bin, c] into acc[argmax[row, bin, c], c] bin by bin.  So each element sums its contributions in ascending
// (row, ph, pw) order -- the loop order of torchvision's CPU roi_pool backward -- with no atomics and no bank conflicts.
// The tile is then added into grad_in frame (f / roi_T) * feat_T + t_start + f % roi_T with 16-byte accesses; frames
// without a ROI are not touched.
constexpr int kPoolBwdMaxChunk = 64;           // the smallest chunk and the shared-memory budget: common.cuh
constexpr int kPoolBwdBins = 16;               // bins whose (argmax, gradient) loads are in flight together

template <typename T>
__global__ void __launch_bounds__(kPoolBwdMaxChunk) roi_pool_bwd_slice_nhwc_kernel(const T* __restrict__ grad_out, int out_ld,
                                                                                   const int32_t* __restrict__ argmax,
                                                                                   const float* __restrict__ rois, int R, int nbins,
                                                                                   int npix, int C, int roi_T, int feat_T, int t_start,
                                                                                   float* __restrict__ grad_in, int in_ld) {
  extern __shared__ float acc[];                // [npix][chunk]
  __shared__ int rows[kPoolBwdMaxChunk];
  __shared__ int warp_rows[kPoolBwdMaxChunk / 32];
  const int chunk = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = (chunk + 31) >> 5;
  const unsigned mask = chunk >= 32 ? 0xffffffffu : (1u << chunk) - 1u;
  const int f = blockIdx.x, c0 = blockIdx.y * chunk, c = c0 + tid;
  for (int i = tid; i < npix * chunk; i += chunk) acc[i] = 0.0f;
  int seen = 0;                                 // rows of frame f so far (uniform across the CTA)
  for (int base = 0; base < R; base += chunk) {
    const int r = base + tid;
    const bool keep = r < R && (int)rois[5 * (size_t)r] == f;
    const unsigned bal = __ballot_sync(mask, keep);
    __syncthreads();                            // the previous batch's rows have been consumed
    if (lane == 0) warp_rows[warp] = __popc(bal);
    __syncthreads();
    int off = 0, n = 0;
    for (int w = 0; w < nwarps; ++w) { off += w < warp ? warp_rows[w] : 0; n += warp_rows[w]; }
    if (keep) rows[off + __popc(bal & ((1u << lane) - 1u))] = r;
    __syncthreads();
    seen += n;
    if (c >= C) continue;
    for (int j = 0; j < n; ++j) {
      const int row = rows[j];
      const T* g = grad_out + (size_t)row * nbins * out_ld + c;
      const int32_t* a = argmax + (size_t)row * nbins * C + c;
      for (int b0 = 0; b0 < nbins; b0 += kPoolBwdBins) {
        int av[kPoolBwdBins];
        float gv[kPoolBwdBins];
#pragma unroll
        for (int k = 0; k < kPoolBwdBins; ++k) {
          const bool in = b0 + k < nbins;
          av[k] = in ? a[(size_t)(b0 + k) * C] : -1;
          gv[k] = in ? to_f32<T>(g[(size_t)(b0 + k) * out_ld]) : 0.0f;
        }
#pragma unroll
        for (int k = 0; k < kPoolBwdBins; ++k)
          if ((unsigned)av[k] < (unsigned)npix) {   // -1: empty bin, no contribution
            float* s = acc + av[k] * chunk + tid;
            *s = __fadd_rn(*s, gv[k]);
          }
      }
    }
  }
  if (seen == 0) return;
  __syncthreads();
  float* dst = grad_in + ((size_t)(f / roi_T) * feat_T + t_start + f % roi_T) * npix * in_ld + c0;
  const int nv = min(chunk, C - c0) / 4;
  for (int i = tid; i < npix * nv; i += chunk) {
    const int p = i / nv, v = i - p * nv;
    const float4 s = *reinterpret_cast<const float4*>(acc + p * chunk + v * 4);
    float4* d = reinterpret_cast<float4*>(dst + (size_t)p * in_ld + v * 4);
    float4 cur = *d;
    cur.x = __fadd_rn(cur.x, s.x); cur.y = __fadd_rn(cur.y, s.y); cur.z = __fadd_rn(cur.z, s.z); cur.w = __fadd_rn(cur.w, s.w);
    *d = cur;
  }
}

// ---- context-feature gradient (train.py:317-321: temp_context_feat[p] = context_feat[clip(p), :, t_start:t_start+T_len]) --
// dctx[r, c] is the gradient of tube r's context input of the classifier (the slice mean the forward feeds to global_cls).
// acc[b, t, c] += (sum over the tubes r of clip b, ascending r, of dctx[r, c]) / T_len for t in [t_start, t_start + T_len);
// clip(r) = floor(frame(r) / T_len) with frame(r) = tubes[r, 0, 0].  One thread per (clip, channel): no atomics.
// DROP: the classifier read the dropped context (two_branch.py:244), so tube r's term on frame t is multiplied by the factor of
// its element (r, t, c) of the draw (map: DropMap at(r, t, 0, c)), and every frame has its own sum.
template <bool DROP>
__global__ void __launch_bounds__(256) ctx_grad_reduce_kernel(const float* __restrict__ dctx, int dctx_ld, const float* __restrict__ tubes,
                                                              int R, int T_len, int B, int feat_T, int t_start, int C,
                                                              float* __restrict__ acc, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C) return;
  const int b = (int)(i / C), c = (int)(i - (long long)b * C);
  float* d = acc + ((size_t)b * feat_T + t_start) * C + c;
  if constexpr (DROP) {
    for (int t = 0; t < T_len; ++t) {
      float s = 0.0f;
      for (int r = 0; r < R; ++r)
        if ((int)__fdiv_rn(tubes[(size_t)r * T_len * 5], (float)T_len) == b)
          s = __fadd_rn(s, __fmul_rn(dctx[(size_t)r * dctx_ld + c], drop_factor(dd, mp.at(r, t, 0, c))));
      d[(size_t)t * C] = __fadd_rn(d[(size_t)t * C], __fdiv_rn(s, (float)T_len));
    }
  } else {
    float s = 0.0f;
    for (int r = 0; r < R; ++r)
      if ((int)__fdiv_rn(tubes[(size_t)r * T_len * 5], (float)T_len) == b) s = __fadd_rn(s, dctx[(size_t)r * dctx_ld + c]);
    const float v = __fdiv_rn(s, (float)T_len);
    for (int t = 0; t < T_len; ++t) d[(size_t)t * C] = __fadd_rn(d[(size_t)t * C], v);
  }
}

// ---- dropout (two_branch.py:244, 261; the draw itself is dropout.cuh) -------------------------------------------------------
// the keep mask of a whole draw, in the order of the dropped tensor's elements
__global__ void __launch_bounds__(256) dropout_mask_kernel(DropDraw dd, long long n, uint8_t* __restrict__ mask) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    mask[e] = drop_keep(dd, e) ? 1 : 0;
}

// y[m, c] = x[m, c] * factor (fp32 product, rounded once to T) over pixels m = (r * T_len + t) * P + p of a channels-last
// [R, T_len, P, C] slice; element (r, t, p, c) of the draw is mp.at(r, t, p, c).
template <typename T>
__global__ void __launch_bounds__(256) dropout_copy_kernel(const T* __restrict__ x, int x_ld, long long M, int T_len, int P, int C,
                                                           T* __restrict__ y, int y_ld, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long m = i / C;
  const int c = (int)(i - m * C);
  const long long f = m / P;
  const int p = (int)(m - f * P);
  const long long r = f / T_len;
  const int t = (int)(f - r * T_len);
  y[(size_t)m * y_ld + c] = from_f32<T>(__fmul_rn(to_f32<T>(x[(size_t)m * x_ld + c]), drop_factor(dd, mp.at(r, t, p, c))));
}

// out[r, k] = (sum over t ascending of ctx[row(r) * row_stride + t * t_stride + k * k_stride] * factor) / T_len: the temporal
// mean of tube r's dropped context columns (the classifier is linear, so it takes the mean instead of the frames);
// row(r) = row_map[r], or r without a map.  Element (r, t, k) of the draw is mp.at(r, t, 0, k).
__global__ void __launch_bounds__(256) ctx_mean_dropout_kernel(const float* __restrict__ ctx, const int32_t* __restrict__ row_map,
                                                               long long row_stride, int t_stride, int k_stride, int R, int T_len,
                                                               int K, float* __restrict__ out, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)R * K) return;
  const int r = (int)(i / K), k = (int)(i - (long long)r * K);
  const float* src = ctx + (size_t)(row_map ? row_map[r] : r) * row_stride + (size_t)k * k_stride;
  float s = 0.0f;
  for (int t = 0; t < T_len; ++t) s = __fadd_rn(s, __fmul_rn(src[(size_t)t * t_stride], drop_factor(dd, mp.at(r, t, 0, k))));
  out[i] = __fdiv_rn(s, (float)T_len);
}

// ---- small-N linear backward -----------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) linear_bwd_dw_kernel(const T* __restrict__ x, int x_ld, const float* __restrict__ dy,
                                                            int M, int K, int Nn, float* __restrict__ dw,
                                                            float* __restrict__ db) {
  // dw[n][k] = sum_m dy[m][n] * x[m][k]   (m ascending: fixed order);  db[n] = sum_m dy[m][n]
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (long long)Nn * K) {
    const int n = (int)(i / K), k = (int)(i - (long long)n * K);
    float acc = 0.0f;
    for (int m = 0; m < M; ++m) acc = fmaf(dy[(size_t)m * Nn + n], to_f32<T>(x[(size_t)m * x_ld + k]), acc);
    dw[i] = acc;
  }
  if (db && i < Nn) {
    float acc = 0.0f;
    for (int m = 0; m < M; ++m) acc += dy[(size_t)m * Nn + (int)i];
    db[i] = acc;
  }
}

__global__ void __launch_bounds__(256) linear_bwd_dx_kernel(const float* __restrict__ dy, const float* __restrict__ w, int M,
                                                            int K, int Nn, float* __restrict__ dx, int accumulate) {
  // dx[m][k] (+)= sum_n dy[m][n] * w[n][k]
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * K) return;
  const int m = (int)(i / K), k = (int)(i - (long long)m * K);
  float acc = accumulate ? dx[i] : 0.0f;
  for (int n = 0; n < Nn; ++n) acc = fmaf(dy[(size_t)m * Nn + n], w[(size_t)n * K + k], acc);
  dx[i] = acc;
}


// ---- elementwise pieces of the conv backward ---------------------------------------------------------------------------
// y = relu(scale * conv + shift (+ residual))  (Unit3Dpy, i3dpt.py:103-111; Bottleneck, two_branch.py:60-111):
//   dz = dy * [y > 0] * scale      gradient w.r.t. the raw convolution output (operand of dgrad / wgrad)
//   dres += dy * [y > 0]           gradient flowing into the residual input, accumulated in place
// dy / y / dres are channel slices of wider buffers of T (fp16 or fp32; ld, coff); dz is dense [M, C] at dz_ld / dz_coff.
// One thread per 16-byte vector (8 fp16 or 4 fp32 channels).
template <typename T>
__global__ void __launch_bounds__(256) act_bwd_kernel(const T* __restrict__ dy, int dy_ld, const T* __restrict__ y,
                                                      int y_ld, const float* __restrict__ scale, int relu, long long M, int C,
                                                      T* __restrict__ dz, int dz_ld, T* __restrict__ dres,
                                                      int dres_ld) {
  constexpr int V = Vec16<T>::N, LOG_V = V == 8 ? 3 : 2;
  const int cv = C >> LOG_V;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * cv) return;
  const long long m = i / cv;
  const int c = (int)(i - m * cv) * V;
  float g[V], v[V];
  load16(dy + (size_t)m * dy_ld + c, g);
  if (relu) {
    load16(y + (size_t)m * y_ld + c, v);
#pragma unroll
    for (int k = 0; k < V; ++k) g[k] = v[k] > 0.0f ? g[k] : 0.0f;
  }
  if (dres) {
    float r[V];
    load16(dres + (size_t)m * dres_ld + c, r);
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] += g[k];
    store16(dres + (size_t)m * dres_ld + c, r);
  }
  if (scale) {
#pragma unroll
    for (int k = 0; k < V; ++k) g[k] *= scale[c + k];
  }
  store16(dz + (size_t)m * dz_ld + c, g);
}

// column sums of a [M, C] fp16 / fp32 matrix in fp32 (bias gradients), fixed order: thread per column block, rows ascending
// in chunks that a second pass adds in chunk order
template <typename T>
__global__ void __launch_bounds__(256) colsum_partial_kernel(const T* __restrict__ x, int ld, long long M, int C, int rows_per,
                                                             float* __restrict__ partial) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long m0 = (long long)blockIdx.y * rows_per, m1 = m0 + rows_per < M ? m0 + rows_per : M;
  float acc = 0.0f;
  for (long long m = m0; m < m1; ++m) acc += to_f32<T>(x[(size_t)m * ld + c]);
  partial[(size_t)blockIdx.y * C + c] = acc;
}
__global__ void __launch_bounds__(256) colsum_reduce_kernel(const float* __restrict__ partial, int chunks, int C, float scale,
                                                            float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.0f;
  for (int k = 0; k < chunks; ++k) acc += partial[(size_t)k * C + c];
  out[c] = acc * scale;
}

// temporal-mean backward (two_branch.py:249: the class scores are averaged over T'):  dx[a][b][p][c] += g[a][p*C + c] / B
// DROP: the mean was taken over the dropped frames, so each term is also multiplied by the factor of element mp.at(a, b, p, c)
// of the draw.
template <typename T, bool DROP>
__global__ void __launch_bounds__(256) mean_mid_bwd_kernel(const float* __restrict__ g, int A, int B, int P, int C, float gscale,
                                                           T* __restrict__ dx, int ld, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)A * B * P * C) return;
  const int c = (int)(i % C);
  long long r = i / C;
  const int p = (int)(r % P); r /= P;
  const int b = (int)(r % B);
  const int a = (int)(r / B);
  T* d = dx + ((((size_t)a * B + b) * P + p) * ld + c);
  float v = g[(size_t)a * P * C + (size_t)p * C + c] * gscale / (float)B;
  if constexpr (DROP) v = v * drop_factor(dd, mp.at(a, b, p, c));
  *d = from_f32<T>(to_f32<T>(*d) + v);
}

// fp32 [M, C] (scaled) accumulated into an fp16 channel slice.  DROP: src is the gradient of the dropped copy of the slice,
// whose pixel m = f * P + p, channel c is element mp.at(f, 0, p, c) of the draw.
template <bool DROP>
__global__ void __launch_bounds__(256) f32_accum_f16_kernel(const float* __restrict__ src, long long M, int C, float gscale,
                                                            __half* __restrict__ dst, int ld, int P, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long m = i / C;
  const int c = (int)(i - m * C);
  __half* d = dst + (size_t)m * ld + c;
  float v = src[i];
  if constexpr (DROP) v = v * drop_factor(dd, mp.at(m / P, 0, (int)(m % P), c));
  *d = __float2half_rn(__half2float(*d) + v * gscale);
}

// the same into an fp32 channel slice (the fp32 training path)
template <bool DROP>
__global__ void __launch_bounds__(256) f32_accum_f32_kernel(const float* __restrict__ src, long long M, int C, float gscale,
                                                            float* __restrict__ dst, int ld, int P, DropDraw dd, DropMap mp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long m = i / C;
  const int c = (int)(i - m * C);
  float* d = dst + (size_t)m * ld + c;
  float v = src[i];
  if constexpr (DROP) v = v * drop_factor(dd, mp.at(m / P, 0, (int)(m % P), c));
  *d = *d + v * gscale;
}

// ---- max-pool backward (MaxPool3dTFPadding, i3dpt.py:114-126: zero ConstantPad3d, then MaxPool3d) ---------------------------
// Pass 1 (per output): which tap of the window holds the maximum -- first maximum in (kt, kh, kw) scan order with '>' like
// ATen's max_pool3d_with_indices; a padded position holds the value 0 and takes part (its gradient is dropped).
// Pass 2 (per input): gather dy from the windows whose recorded tap points at this input.  No atomics.
struct PoolGeom { int N, T, H, W, C, KT, KH, KW, ST, SH, SW, PT, PH, PW, OT, OH, OW, QT, QH, QW; };   // Q*: high-side zero padding

template <typename T>
__global__ void __launch_bounds__(256) maxpool_argmax_kernel(PoolGeom g, const T* __restrict__ x, int x_ld,
                                                             uint8_t* __restrict__ arg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)g.N * g.OT * g.OH * g.OW * g.C;
  if (i >= total) return;
  const int c = (int)(i % g.C);
  long long r = i / g.C;
  const int ow = (int)(r % g.OW); r /= g.OW;
  const int oh = (int)(r % g.OH); r /= g.OH;
  const int ot = (int)(r % g.OT);
  const int n = (int)(r / g.OT);
  float best = 0.0f;
  int bi = -1, tap = 0;
  for (int kt = 0; kt < g.KT; ++kt)
    for (int kh = 0; kh < g.KH; ++kh)
      for (int kw = 0; kw < g.KW; ++kw, ++tap) {
        const int t = ot * g.ST + kt - g.PT, h = oh * g.SH + kh - g.PH, w = ow * g.SW + kw - g.PW;
        // positions beyond the padded extent do not exist (ceil_mode overhang); inside the pad the value is 0
        const bool in_t = t >= 0 && t < g.T, in_h = h >= 0 && h < g.H, in_w = w >= 0 && w < g.W;
        const bool pad_t = t < 0 || (t >= g.T && t < g.T + g.QT), pad_h = h < 0 || (h >= g.H && h < g.H + g.QH),
                   pad_w = w < 0 || (w >= g.W && w < g.W + g.QW);
        if (!((in_t || pad_t) && (in_h || pad_h) && (in_w || pad_w))) continue;
        const bool real = in_t && in_h && in_w;
        const float v = real ? to_f32<T>(x[((((size_t)n * g.T + t) * g.H + h) * g.W + w) * x_ld + c]) : 0.0f;
        if (bi < 0 || v > best) { best = v; bi = real ? tap : 254; }
      }
  arg[i] = (uint8_t)(bi < 0 ? 255 : bi);
}

template <typename T>
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(PoolGeom g, const T* __restrict__ dy, int dy_ld,
                                                          const uint8_t* __restrict__ arg, T* __restrict__ dx, int dx_ld) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)g.N * g.T * g.H * g.W * g.C;
  if (i >= total) return;
  const int c = (int)(i % g.C);
  long long r = i / g.C;
  const int w = (int)(r % g.W); r /= g.W;
  const int h = (int)(r % g.H); r /= g.H;
  const int t = (int)(r % g.T);
  const int n = (int)(r / g.T);
  float acc = 0.0f;
  // windows (ot, oh, ow) with ot*ST + kt - PT == t  ->  kt = t + PT - ot*ST in [0, KT)
  for (int kt = 0; kt < g.KT; ++kt) {
    const int tn = t + g.PT - kt;
    if (tn < 0 || tn % g.ST) continue;
    const int ot = tn / g.ST;
    if (ot >= g.OT) continue;
    for (int kh = 0; kh < g.KH; ++kh) {
      const int hn = h + g.PH - kh;
      if (hn < 0 || hn % g.SH) continue;
      const int oh = hn / g.SH;
      if (oh >= g.OH) continue;
      for (int kw = 0; kw < g.KW; ++kw) {
        const int wn = w + g.PW - kw;
        if (wn < 0 || wn % g.SW) continue;
        const int ow = wn / g.SW;
        if (ow >= g.OW) continue;
        const size_t o = (((size_t)n * g.OT + ot) * g.OH + oh) * g.OW + ow;
        if (arg[o * g.C + c] == (uint8_t)((kt * g.KH + kh) * g.KW + kw)) acc += to_f32<T>(dy[o * dy_ld + c]);
      }
    }
  }
  T* d = dx + ((((size_t)n * g.T + t) * g.H + h) * g.W + w) * dx_ld + c;
  *d = from_f32<T>(to_f32<T>(*d) + acc);
}

// ---- 1x1 convolution weight gradient on the tensor cores ------------------------------------------------------------
// dW[co][ci] = sum_m dz[m][co] * x[m][ci].  A CTA owns a 64 (co) x 64 (ci) tile of dW and one chunk of kWgChunk pixels;
// both operands are staged [32 pixels][64 channels] in shared memory and fed to wmma (fp16 x fp16 -> fp32) as A^T
// (column-major: element (co, m) at m * ld + co) and B (row-major: element (m, ci) at m * ld + ci).  The per-chunk
// partial tiles are summed by a second kernel in chunk order (deterministic), which also applies `scale`.
constexpr int kWgTile = 64, kWgPix = 32, kWgChunk = 2048;

// Filters larger than 1x1x1 (stride 1): tap (kt, kh, kw) pairs output pixel (n, t, h, w) with input pixel
// (t + kt - PT, h + kh - PH, w + kw - PW), zero outside the map (the TF-"SAME" padding, i3dpt.py:14-31); blockIdx.y also
// enumerates the taps and the staging of x applies the shift.
struct WgGeom { int T, H, W, KT, KH, KW, PT, PH, PW, taps; };

__global__ void __launch_bounds__(128) conv1x1_wgrad_partial_kernel(const __half* __restrict__ dz, int dz_ld,
                                                                    const __half* __restrict__ x, int x_ld, int M, int Cout,
                                                                    int Cin, WgGeom wg, float* __restrict__ partial) {
  using namespace nvcuda;
  __shared__ __align__(32) __half sA[kWgPix][kWgTile + 8];
  __shared__ __align__(32) __half sB[kWgPix][kWgTile + 8];
  const int tiles_ci = gridDim.y / wg.taps;
  const int tap = blockIdx.y / tiles_ci;
  const int co0 = blockIdx.x * kWgTile, ci0 = (blockIdx.y - tap * tiles_ci) * kWgTile, chunk = blockIdx.z;
  const int dkw = tap % wg.KW - wg.PW, dkh = (tap / wg.KW) % wg.KH - wg.PH, dkt = tap / (wg.KW * wg.KH) - wg.PT;
  const int m_beg = chunk * kWgChunk, m_end = min(M, m_beg + kWgChunk);
  const int warp = threadIdx.x >> 5;                 // 4 warps: warp w owns rows (co) [16 w, 16 w + 16) x all 64 ci
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) wmma::fill_fragment(acc[j], 0.0f);
  for (int m0 = m_beg; m0 < m_end; m0 += kWgPix) {
    // stage 32 pixels x 64 channels of each operand (16-byte vectors; rows past M and channels past C read as zero)
    for (int i = threadIdx.x; i < kWgPix * (kWgTile / 8); i += blockDim.x) {
      const int r = i / (kWgTile / 8), v = i - r * (kWgTile / 8);
      const int m = m0 + r;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (m < m_end) {
        if (co0 + v * 8 < Cout) a = *reinterpret_cast<const uint4*>(dz + (size_t)m * dz_ld + co0 + v * 8);
        long long src = m;
        bool ok = true;
        if (wg.taps > 1) {
          const int w = m % wg.W, h = (m / wg.W) % wg.H, t = (m / (wg.W * wg.H)) % wg.T;
          const int ws = w + dkw, hs = h + dkh, ts = t + dkt;
          ok = ws >= 0 && ws < wg.W && hs >= 0 && hs < wg.H && ts >= 0 && ts < wg.T;
          src = (long long)m + ((long long)dkt * wg.H + dkh) * wg.W + dkw;
        }
        if (ok && ci0 + v * 8 < Cin) b = *reinterpret_cast<const uint4*>(x + (size_t)src * x_ld + ci0 + v * 8);
      }
      *reinterpret_cast<uint4*>(&sA[r][v * 8]) = a;
      *reinterpret_cast<uint4*>(&sB[r][v * 8]) = b;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kWgPix; kk += 16) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::col_major> fa;   // A(co, m) = sA[m][co]
      wmma::load_matrix_sync(fa, &sA[kk][warp * 16], kWgTile + 8);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::row_major> fb;  // B(m, ci) = sB[m][ci]
        wmma::load_matrix_sync(fb, &sB[kk][j * 16], kWgTile + 8);
        wmma::mma_sync(acc[j], fa, fb, acc[j]);
      }
    }
    __syncthreads();
  }
  float* out = partial + ((size_t)chunk * gridDim.x * gridDim.y + (size_t)blockIdx.x * gridDim.y + blockIdx.y) * (kWgTile * kWgTile);   // [chunk][co tile][tap][ci tile]
#pragma unroll
  for (int j = 0; j < 4; ++j) wmma::store_matrix_sync(out + (warp * 16) * kWgTile + j * 16, acc[j], kWgTile, wmma::mem_row_major);
}

// partial tiles are laid out [chunk][co tile][tap][ci tile][64 x 64]; dw is [Cout][taps][dw_ld >= Cin]
__global__ void __launch_bounds__(256) conv1x1_wgrad_reduce_kernel(const float* __restrict__ partial, int chunks, int tiles_co,
                                                                   int tiles_ci, int taps, int Cout, int Cin, float scale,
                                                                   float* __restrict__ dw, int dw_ld, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Cout * taps * Cin) return;
  const int ci = (int)(i % Cin);
  const int tap = (int)((i / Cin) % taps);
  const int co = (int)(i / ((long long)Cin * taps));
  const int tco = co / kWgTile, tci = ci / kWgTile;
  const size_t off = (((size_t)tco * taps + tap) * tiles_ci + tci) * (kWgTile * kWgTile) + (size_t)(co - tco * kWgTile) * kWgTile + (ci - tci * kWgTile);
  const size_t stride = (size_t)tiles_co * taps * tiles_ci * (kWgTile * kWgTile);
  float acc = 0.0f;
  for (int c = 0; c < chunks; ++c) acc += partial[off + (size_t)c * stride];   // chunk order: deterministic
  float* d = dw + ((size_t)co * taps + tap) * dw_ld + ci;
  *d = accumulate ? *d + acc * scale : acc * scale;
}


// ---- fp32 weight gradient of a 3-D convolution on the CUDA cores (the fp32 training path) ---------------------------
// dW[co][tap][ci] = sum_m dz[m][co] * x[src(m, tap)][ci] over the output pixels m = (n, ot, oh, ow), where tap (kt, kh, kw)
// reads input pixel (n, ot * ST + kt - PT, oh * SH + kh - PH, ow * SW + kw - PW) of the [N, T, H, W] input, zero outside
// it (the TF-"SAME" padding, i3dpt.py:14-31, with its high side implied by the output extent).  As a GEMM: rows co,
// columns j = tap * Cin + ci (Cin % 4 == 0, so the 4 columns of a vector share a tap), reduction over m.  Folding the taps
// into the columns keeps thin inputs such as the fp32 stem (Cin = 4, 343 taps) as dense as wide ones.
// A CTA owns a 64 (co) x 64 (j) tile for one chunk of pixels: 16 pixels of both operands are staged per step in shared
// memory (double-buffered, the next step's 16-byte loads in flight during the current FFMAs), and each of the 256 threads
// accumulates a 4 x 4 register tile with fmaf -- fp32 FFMA throughout, no TF32.  Partial tiles land in the workspace and a
// second kernel adds them in chunk order, so the result is bit-identical from run to run.
constexpr int kWfTile = 64, kWfStep = 16;
constexpr int kWfTargetCtas = 2048;   // chunks per tile are chosen for about this many CTAs (a shape-only rule: deterministic)
constexpr int kWfMinChunk = 256;      // pixels

struct WfGeom {
  int T, H, W, OT, OH, OW, KH, KW, ST, SH, SW, PT, PH, PW;
  int Cin, cols;                      // cols = taps * Cin
  int M, chunk;                       // output pixels, pixels per chunk (a multiple of kWfStep)
};

__global__ void __launch_bounds__(256) conv_wgrad_f32_partial_kernel(const float* __restrict__ dz, int dz_ld,
                                                                     const float* __restrict__ x, int x_ld, int Cout, WfGeom g,
                                                                     float* __restrict__ partial) {
  __shared__ __align__(16) float sA[2][kWfStep][kWfTile + 4];   // sA[k][co]
  __shared__ __align__(16) float sB[2][kWfStep][kWfTile + 4];   // sB[k][j]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;    // compute: co ty*4.., j tx*4..
  const int lr = tid >> 4, lv = tid & 15;                       // staging: pixel row lr, 4-channel vector lv
  const int co0 = blockIdx.x * kWfTile, j0 = blockIdx.y * kWfTile;
  const int m_beg = blockIdx.z * g.chunk, m_end = min(g.M, m_beg + g.chunk);
  const int co_l = co0 + lv * 4, j_l = j0 + lv * 4;
  const bool a_ok = co_l < Cout, b_ok = j_l < g.cols;
  int dkt = 0, dkh = 0, dkw = 0, ci = 0;
  if (b_ok) {
    const int tap = j_l / g.Cin;
    ci = j_l - tap * g.Cin;
    dkw = tap % g.KW - g.PW;
    dkh = (tap / g.KW) % g.KH - g.PH;
    dkt = tap / (g.KW * g.KH) - g.PT;
  }
  float4 ra, rb;
  auto load = [&](int m0) {
    const int m = m0 + lr;
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    rb = ra;
    if (m >= m_end) return;
    if (a_ok) ra = *reinterpret_cast<const float4*>(dz + (size_t)m * dz_ld + co_l);
    if (b_ok) {
      const int ow = m % g.OW, r1 = m / g.OW, oh = r1 % g.OH, r2 = r1 / g.OH, ot = r2 % g.OT, n = r2 / g.OT;
      const int it = ot * g.ST + dkt, ih = oh * g.SH + dkh, iw = ow * g.SW + dkw;
      if (it >= 0 && it < g.T && ih >= 0 && ih < g.H && iw >= 0 && iw < g.W)
        rb = *reinterpret_cast<const float4*>(x + ((((size_t)n * g.T + it) * g.H + ih) * g.W + iw) * x_ld + ci);
    }
  };
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  load(m_beg);
  int buf = 0;
  for (int m0 = m_beg; m0 < m_end; m0 += kWfStep) {
    // one barrier per step: the buffer written here was last read two steps ago, before the previous barrier
    *reinterpret_cast<float4*>(&sA[buf][lr][lv * 4]) = ra;
    *reinterpret_cast<float4*>(&sB[buf][lr][lv * 4]) = rb;
    __syncthreads();
    if (m0 + kWfStep < m_end) load(m0 + kWfStep);
#pragma unroll
    for (int k = 0; k < kWfStep; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&sA[buf][k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&sB[buf][k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    buf ^= 1;
  }
  // partial tiles [chunk][j tile][co tile][64 x 64]
  float* out = partial + (((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * (kWfTile * kWfTile);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(out + (ty * 4 + i) * kWfTile + tx * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}

// dw[co][tap][ci] (dw_ld >= Cin) = scale * (sum of the chunks' partial tiles in chunk order) (+ dw when accumulate)
__global__ void __launch_bounds__(256) conv_wgrad_f32_reduce_kernel(const float* __restrict__ partial, int chunks, int tiles_co,
                                                                    int tiles_j, int Cout, int Cin, int cols, float scale,
                                                                    float* __restrict__ dw, int dw_ld, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Cout * cols) return;
  const int co = (int)(i / cols), j = (int)(i - (long long)co * cols);
  const int tco = co / kWfTile, tj = j / kWfTile;
  const size_t off = ((size_t)tj * tiles_co + tco) * (kWfTile * kWfTile) + (size_t)(co - tco * kWfTile) * kWfTile + (j - tj * kWfTile);
  const size_t stride = (size_t)tiles_co * tiles_j * (kWfTile * kWfTile);
  float acc = 0.0f;
  for (int c = 0; c < chunks; ++c) acc += partial[off + (size_t)c * stride];
  const int tap = j / Cin, ci = j - tap * Cin;
  const int taps = cols / Cin;
  float* d = dw + ((size_t)co * taps + tap) * dw_ld + ci;
  *d = accumulate ? *d + acc * scale : acc * scale;
}

// The chunk plan of step_conv_wgrad_f32: a function of the shape alone, so that the summation order does not depend on
// the device.
struct WfPlan { int tiles_co, tiles_j, chunks, chunk; };
inline WfPlan wgrad_f32_plan(long long M, int Cout, long long cols) {
  WfPlan p;
  p.tiles_co = ceil_div(Cout, kWfTile);
  p.tiles_j = ceil_div(cols, kWfTile);
  const long long tiles = (long long)p.tiles_co * p.tiles_j;
  long long want = (kWfTargetCtas + tiles - 1) / tiles;
  const long long most = (M + kWfMinChunk - 1) / kWfMinChunk;
  want = want < 1 ? 1 : (want > most ? most : want);
  const long long per = (M + want - 1) / want;
  p.chunk = (int)((per + kWfStep - 1) / kWfStep * kWfStep);
  p.chunks = ceil_div(M, p.chunk);
  return p;
}

}  // namespace step

using namespace step;

extern "C" int step_head_losses_f32(const float* logits, const float* local_loc, const float* first_loc, const float* last_loc,
                                    const float* tubes, const float* targets, int N, int cls, int T_len, int T, int Tc, float w_loc,
                                    float w_nb, float* loss_cls, float* loss_loc, float* loss_nb, int* flags, float* dlogits,
                                    float* dloc, float* dfirst, float* dlast, float* scratch, step_stream_t stream) {
  STEP_CHECK_ARG(N > 0 && cls > 0 && T > 0 && T_len >= T && T_len % T == 0, "head_losses: bad shape N=%d cls=%d T'=%d T=%d", N, cls, T_len, T);
  STEP_CHECK_ARG(logits && local_loc && first_loc && last_loc && tubes && targets && loss_cls && loss_loc && loss_nb && flags && scratch,
                 "head_losses: null pointer");
  STEP_CHECK_ARG((dfirst == nullptr) == (dlast == nullptr), "head_losses: dfirst / dlast go together");
  LossGeom g;
  const int chunks = T_len / T;
  g.N = N; g.cls = cls; g.T_len = T_len; g.Tc = Tc; g.half_T = T / 2;   // Tc = frames of first_loc / last_loc (python slice clipping)
  g.first_idx = T / 2; g.last_idx = (chunks - 1) * T + T / 2; g.centre = (chunks / 2) * T + T / 2;   // two_branch.py:226-228
  g.s0 = g.first_idx - g.half_T; g.e0 = g.last_idx - g.half_T;
  g.tgt_ld = 6 + cls; g.w_loc = w_loc; g.w_nb = w_nb;
  STEP_CHECK_ARG(Tc > g.half_T && g.s0 >= 0 && g.s0 + Tc <= T_len && g.e0 + Tc <= T_len, "head_losses: chunk slices out of range");
  head_losses_kernel<<<1, 256, 0, cu(stream)>>>(g, logits, local_loc, first_loc, last_loc, tubes, targets, loss_cls, loss_loc, loss_nb,
                                                flags, dlogits, dloc, dfirst, dlast, scratch);
  STEP_LAUNCH_CHECK("head_losses_kernel");
  return 0;
}

extern "C" int step_cls_loss_f32(const float* logits, const float* targets, int N, int cls, float* loss_cls, int* flags,
                                 float* dlogits, step_stream_t stream) {
  STEP_CHECK_ARG(N > 0 && cls > 0, "cls_loss: bad shape N=%d cls=%d", N, cls);
  STEP_CHECK_ARG(logits && targets && loss_cls && flags, "cls_loss: null pointer");
  cls_loss_kernel<<<1, 256, 0, cu(stream)>>>(N, cls, logits, targets, loss_cls, flags, dlogits);
  STEP_LAUNCH_CHECK("cls_loss_kernel");
  return 0;
}

extern "C" int step_roi_align_bwd_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                                       int pw, int K, int H, int W, int C, int sampling_ratio, float* grad_in, int in_ld,
                                       step_stream_t stream) {
  STEP_CHECK_ARG(K > 0 && H > 0 && W > 0 && C > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_bwd_nhwc: bad shape");
  STEP_CHECK_ARG(dtype == STEP_F32 || dtype == STEP_F16, "roi_align_bwd_nhwc: bad dtype");
  STEP_CHECK_ARG(C % 4 == 0 && in_ld % 4 == 0 && out_ld % 4 == 0 && in_ld >= C && out_ld >= C, "roi_align_bwd_nhwc: C / ld must be multiples of 4");
  STEP_CHECK_ARG(grad_in && (R == 0 || (grad_out && rois)), "roi_align_bwd_nhwc: null pointer");
  STEP_CHECK_ARG((((uintptr_t)grad_in | (uintptr_t)grad_out) & 15) == 0, "roi_align_bwd_nhwc: pointers must be 16-byte aligned");
  if (dtype == STEP_F32)
    roi_align_bwd_nhwc_kernel<float><<<K, 256, 0, cu(stream)>>>((const float*)grad_out, out_ld, rois, R, scale, H, W, C, ph, pw,
                                                                 sampling_ratio, grad_in, in_ld);
  else
    roi_align_bwd_nhwc_kernel<__half><<<K, 256, 0, cu(stream)>>>((const __half*)grad_out, out_ld, rois, R, scale, H, W, C, ph, pw,
                                                                  sampling_ratio, grad_in, in_ld);
  STEP_LAUNCH_CHECK("roi_align_bwd_nhwc_kernel");
  return 0;
}

extern "C" size_t step_roi_align_bwd_slice_workspace_bytes(int K, int H, int W, int C, int roi_T, int feat_T) {
  if (K <= 0 || H <= 0 || W <= 0 || C <= 0 || roi_T <= 0 || feat_T <= 0) return 0;
  return (size_t)(K / feat_T) * roi_T * H * W * C * sizeof(float);
}

extern "C" int step_roi_align_bwd_slice_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                                             int pw, int K, int H, int W, int C, int sampling_ratio, int roi_T, int feat_T, int t_start,
                                             float* grad_in, int in_ld, void* workspace, size_t ws_bytes, step_stream_t stream) {
  STEP_CHECK_ARG(K > 0 && H > 0 && W > 0 && C > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_bwd_slice_nhwc: bad shape");
  STEP_CHECK_ARG(dtype == STEP_F32 || dtype == STEP_F16, "roi_align_bwd_slice_nhwc: bad dtype");
  STEP_CHECK_ARG(C % 4 == 0 && in_ld % 4 == 0 && out_ld % 4 == 0 && in_ld >= C && out_ld >= C,
                 "roi_align_bwd_slice_nhwc: C / ld must be multiples of 4");
  STEP_CHECK_ARG(feat_T > 0 && K % feat_T == 0 && roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T,
                 "roi_align_bwd_slice_nhwc: bad frame map roi_T=%d feat_T=%d t_start=%d K=%d", roi_T, feat_T, t_start, K);
  STEP_CHECK_ARG(grad_in && workspace && (R == 0 || (grad_out && rois)), "roi_align_bwd_slice_nhwc: null pointer");
  STEP_CHECK_ARG((((uintptr_t)grad_in | (uintptr_t)grad_out | (uintptr_t)workspace) & 15) == 0,
                 "roi_align_bwd_slice_nhwc: pointers must be 16-byte aligned");
  const size_t need = step_roi_align_bwd_slice_workspace_bytes(K, H, W, C, roi_T, feat_T);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "roi_align_bwd_slice_nhwc: workspace %zu < %zu", ws_bytes, need);
  const int frames = (K / feat_T) * roi_T;
  if (dtype == STEP_F32)
    roi_align_bwd_slice_nhwc_kernel<float><<<frames, 256, 0, cu(stream)>>>((const float*)grad_out, out_ld, rois, R, scale, H, W, C, ph, pw,
                                                                            sampling_ratio, roi_T, feat_T, t_start, (float*)workspace,
                                                                            grad_in, in_ld);
  else
    roi_align_bwd_slice_nhwc_kernel<__half><<<frames, 256, 0, cu(stream)>>>((const __half*)grad_out, out_ld, rois, R, scale, H, W, C, ph,
                                                                             pw, sampling_ratio, roi_T, feat_T, t_start, (float*)workspace,
                                                                             grad_in, in_ld);
  STEP_LAUNCH_CHECK("roi_align_bwd_slice_nhwc_kernel");
  return 0;
}

extern "C" int step_roi_pool_bwd_slice_nhwc(const void* grad_out, int dtype, int out_ld, const int32_t* argmax, const float* rois, int R,
                                            int ph, int pw, int K, int H, int W, int C, int roi_T, int feat_T, int t_start,
                                            float* grad_in, int in_ld, step_stream_t stream) {
  STEP_CHECK_ARG(K > 0 && H > 0 && W > 0 && C > 0 && R >= 0 && ph > 0 && pw > 0, "roi_pool_bwd_slice_nhwc: bad shape");
  STEP_CHECK_ARG(dtype == STEP_F32 || dtype == STEP_F16, "roi_pool_bwd_slice_nhwc: bad dtype");
  STEP_CHECK_ARG(C % 4 == 0 && in_ld % 4 == 0 && in_ld >= C && out_ld >= C,
                 "roi_pool_bwd_slice_nhwc: C=%d in_ld=%d must be multiples of 4, out_ld=%d >= C", C, in_ld, out_ld);
  STEP_CHECK_ARG(feat_T > 0 && K % feat_T == 0 && roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T,
                 "roi_pool_bwd_slice_nhwc: bad frame map roi_T=%d feat_T=%d t_start=%d K=%d", roi_T, feat_T, t_start, K);
  STEP_CHECK_ARG(grad_in && (R == 0 || (grad_out && argmax && rois)), "roi_pool_bwd_slice_nhwc: null pointer");
  STEP_CHECK_ARG(((uintptr_t)grad_in & 15) == 0, "roi_pool_bwd_slice_nhwc: grad_in must be 16-byte aligned");
  const long long npix = (long long)H * W;
  STEP_CHECK_ARG(npix <= kPoolBwdMaxPixels,
                 "roi_pool_bwd_slice_nhwc: H*W=%lld exceeds the %d-pixel limit of the shared-memory accumulator (inputs up to ~1280x1280)",
                 npix, kPoolBwdMaxPixels);
  if (R == 0) return 0;
  // the widest channel chunk whose accumulator fits, no wider than C needs
  int chunk = kPoolBwdMaxChunk;
  while (chunk > kPoolBwdMinChunk && (npix * chunk * (long long)sizeof(float) > kPoolBwdSmem || chunk >= 2 * C)) chunk /= 2;
  const size_t smem = (size_t)npix * chunk * sizeof(float);
  const dim3 grid((K / feat_T) * roi_T, ceil_div(C, chunk));
  static std::atomic<unsigned long long> seen32{0}, seen16{0};
  if (dtype == STEP_F32) {
    if (int rc = allow_dynamic_smem(roi_pool_bwd_slice_nhwc_kernel<float>, seen32, kPoolBwdSmem, "roi_pool_bwd_slice_nhwc")) return rc;
    roi_pool_bwd_slice_nhwc_kernel<float><<<grid, chunk, smem, cu(stream)>>>((const float*)grad_out, out_ld, argmax, rois, R, ph * pw,
                                                                             (int)npix, C, roi_T, feat_T, t_start, grad_in, in_ld);
  } else {
    if (int rc = allow_dynamic_smem(roi_pool_bwd_slice_nhwc_kernel<__half>, seen16, kPoolBwdSmem, "roi_pool_bwd_slice_nhwc")) return rc;
    roi_pool_bwd_slice_nhwc_kernel<__half><<<grid, chunk, smem, cu(stream)>>>((const __half*)grad_out, out_ld, argmax, rois, R, ph * pw,
                                                                              (int)npix, C, roi_T, feat_T, t_start, grad_in, in_ld);
  }
  STEP_LAUNCH_CHECK("roi_pool_bwd_slice_nhwc_kernel");
  return 0;
}

extern "C" int step_ctx_grad_reduce_f32(const float* dctx, int dctx_ld, const float* tubes, int R, int T_len, int B, int feat_T,
                                        int t_start, int C, float* acc, step_stream_t stream) {
  STEP_CHECK_ARG(B > 0 && C > 0 && R >= 0 && T_len > 0 && dctx_ld >= C && t_start >= 0 && t_start + T_len <= feat_T,
                 "ctx_grad_reduce: bad shape B=%d C=%d R=%d T_len=%d feat_T=%d t_start=%d", B, C, R, T_len, feat_T, t_start);
  STEP_CHECK_ARG(acc && (R == 0 || (dctx && tubes)), "ctx_grad_reduce: null pointer");
  ctx_grad_reduce_kernel<false><<<ceil_div((long long)B * C, 256), 256, 0, cu(stream)>>>(dctx, dctx_ld, tubes, R, T_len, B, feat_T,
                                                                                         t_start, C, acc, DropDraw{}, DropMap{});
  STEP_LAUNCH_CHECK("ctx_grad_reduce_kernel");
  return 0;
}

extern "C" int step_linear_small_n_bwd(const void* x, int dtype, int M, int K, int x_ld, const float* w, const float* dy, int Nn,
                                       float* dx, int dx_accumulate, float* dw, float* db, step_stream_t stream) {
  STEP_CHECK_ARG(M > 0 && K > 0 && Nn > 0 && dy, "linear_small_n_bwd: bad arguments");
  STEP_CHECK_ARG(dtype == STEP_F32 || dtype == STEP_F16, "linear_small_n_bwd: bad dtype");
  if (dw) {
    STEP_CHECK_ARG(x != nullptr, "linear_small_n_bwd: dw needs x");
    const long long tot = (long long)Nn * K;
    const int grid = ceil_div(tot, 256);
    if (dtype == STEP_F32) linear_bwd_dw_kernel<float><<<grid, 256, 0, cu(stream)>>>((const float*)x, x_ld, dy, M, K, Nn, dw, db);
    else linear_bwd_dw_kernel<__half><<<grid, 256, 0, cu(stream)>>>((const __half*)x, x_ld, dy, M, K, Nn, dw, db);
    STEP_LAUNCH_CHECK("linear_bwd_dw_kernel");
  }
  if (dx) {
    STEP_CHECK_ARG(w != nullptr, "linear_small_n_bwd: dx needs w");
    linear_bwd_dx_kernel<<<ceil_div((long long)M * K, 256), 256, 0, cu(stream)>>>(dy, w, M, K, Nn, dx, dx_accumulate);
    STEP_LAUNCH_CHECK("linear_bwd_dx_kernel");
  }
  return 0;
}

extern "C" size_t step_conv_wgrad_workspace_bytes(int M, int Cout, int Cin, int taps) {
  const size_t chunks = (size_t)ceil_div(M, kWgChunk), tco = (size_t)ceil_div(Cout, kWgTile), tci = (size_t)ceil_div(Cin, kWgTile);
  return chunks * tco * tci * (size_t)(taps > 0 ? taps : 1) * kWgTile * kWgTile * sizeof(float);
}
extern "C" size_t step_conv1x1_wgrad_workspace_bytes(int M, int Cout, int Cin) { return step_conv_wgrad_workspace_bytes(M, Cout, Cin, 1); }

extern "C" int step_conv1x1_wgrad_f16(const void* dz, int dz_ld, const void* x, int x_ld, int M, int Cout, int Cin, float scale,
                                      float* dw, int dw_ld, int accumulate, void* workspace, size_t ws_bytes,
                                      step_stream_t stream) {
  STEP_CHECK_ARG(M > 0 && Cout > 0 && Cin > 0 && dz && x && dw && workspace, "conv1x1_wgrad: bad arguments");
  STEP_CHECK_ARG(Cout % 8 == 0 && Cin % 8 == 0 && dz_ld % 8 == 0 && x_ld % 8 == 0 && dz_ld >= Cout && x_ld >= Cin && dw_ld >= Cin,
                 "conv1x1_wgrad: channel counts / strides must be multiples of 8");
  STEP_CHECK_ARG((((uintptr_t)dz | (uintptr_t)x) & 15) == 0, "conv1x1_wgrad: pointers must be 16-byte aligned");
  if (ws_bytes < step_conv1x1_wgrad_workspace_bytes(M, Cout, Cin))
    return fail(STEP_E_WORKSPACE, "conv1x1_wgrad: workspace %zu < %zu", ws_bytes, step_conv1x1_wgrad_workspace_bytes(M, Cout, Cin));
  const int chunks = ceil_div(M, kWgChunk), tco = ceil_div(Cout, kWgTile), tci = ceil_div(Cin, kWgTile);
  WgGeom wg = {1, 1, M, 1, 1, 1, 0, 0, 0, 1};
  conv1x1_wgrad_partial_kernel<<<dim3(tco, tci, chunks), 128, 0, cu(stream)>>>((const __half*)dz, dz_ld, (const __half*)x, x_ld, M, Cout,
                                                                               Cin, wg, (float*)workspace);
  STEP_LAUNCH_CHECK("conv1x1_wgrad_partial_kernel");
  conv1x1_wgrad_reduce_kernel<<<ceil_div((long long)Cout * Cin, 256), 256, 0, cu(stream)>>>((const float*)workspace, chunks, tco, tci, 1,
                                                                                            Cout, Cin, scale, dw, dw_ld, accumulate);
  STEP_LAUNCH_CHECK("conv1x1_wgrad_reduce_kernel");
  return 0;
}

extern "C" int step_conv_wgrad_f16(const void* dz, int dz_ld, const void* x, int x_ld, int N, int T, int H, int W, int Cout, int Cin,
                                   int KT, int KH, int KW, int PT, int PH, int PW, float scale, float* dw, int dw_ld, int accumulate,
                                   void* workspace, size_t ws_bytes, step_stream_t stream) {
  const long long M = (long long)N * T * H * W;
  const int taps = KT * KH * KW;
  STEP_CHECK_ARG(M > 0 && M < (1LL << 31) && Cout > 0 && Cin > 0 && taps > 0 && dz && x && dw && workspace, "conv_wgrad: bad arguments");
  STEP_CHECK_ARG(Cout % 8 == 0 && Cin % 8 == 0 && dz_ld % 8 == 0 && x_ld % 8 == 0 && dz_ld >= Cout && x_ld >= Cin && dw_ld >= Cin,
                 "conv_wgrad: channel counts / strides must be multiples of 8");
  STEP_CHECK_ARG((((uintptr_t)dz | (uintptr_t)x) & 15) == 0, "conv_wgrad: pointers must be 16-byte aligned");
  STEP_CHECK_ARG(PT >= 0 && PT < KT && PH >= 0 && PH < KH && PW >= 0 && PW < KW, "conv_wgrad: bad padding");
  if (ws_bytes < step_conv_wgrad_workspace_bytes((int)M, Cout, Cin, taps))
    return fail(STEP_E_WORKSPACE, "conv_wgrad: workspace %zu < %zu", ws_bytes, step_conv_wgrad_workspace_bytes((int)M, Cout, Cin, taps));
  const int chunks = ceil_div(M, kWgChunk), tco = ceil_div(Cout, kWgTile), tci = ceil_div(Cin, kWgTile);
  STEP_CHECK_ARG((long long)tci * taps <= 65535 && chunks <= 65535, "conv_wgrad: grid too large");
  WgGeom wg = {T, H, W, KT, KH, KW, PT, PH, PW, taps};
  conv1x1_wgrad_partial_kernel<<<dim3(tco, tci * taps, chunks), 128, 0, cu(stream)>>>((const __half*)dz, dz_ld, (const __half*)x, x_ld, (int)M,
                                                                                      Cout, Cin, wg, (float*)workspace);
  STEP_LAUNCH_CHECK("conv_wgrad_partial_kernel");
  conv1x1_wgrad_reduce_kernel<<<ceil_div((long long)Cout * taps * Cin, 256), 256, 0, cu(stream)>>>((const float*)workspace, chunks, tco, tci,
                                                                                                   taps, Cout, Cin, scale, dw, dw_ld, accumulate);
  STEP_LAUNCH_CHECK("conv_wgrad_reduce_kernel");
  return 0;
}

template <typename T>
static int act_bwd_launch(const void* dy, int dy_ld, const void* y, int y_ld, const float* scale, int relu, long long M, int C,
                          void* dz, int dz_ld, void* dres, int dres_ld, step_stream_t stream) {
  constexpr int V = Vec16<T>::N;
  STEP_CHECK_ARG(M > 0 && C > 0 && C % V == 0 && dy_ld % V == 0 && dz_ld % V == 0 && dy && dz && (!relu || (y && y_ld % V == 0)) &&
                 (!dres || dres_ld % V == 0), "act_bwd: bad arguments");
  STEP_CHECK_ARG((((uintptr_t)dy | (uintptr_t)y | (uintptr_t)dz | (uintptr_t)dres) & 15) == 0, "act_bwd: pointers must be 16-byte aligned");
  act_bwd_kernel<T><<<ceil_div(M * (C / V), 256), 256, 0, cu(stream)>>>((const T*)dy, dy_ld, (const T*)y, y_ld, scale, relu, M, C,
                                                                        (T*)dz, dz_ld, (T*)dres, dres_ld);
  STEP_LAUNCH_CHECK("act_bwd_kernel");
  return 0;
}

extern "C" int step_act_bwd_f16(const void* dy, int dy_ld, const void* y, int y_ld, const float* scale, int relu, long long M, int C,
                                void* dz, int dz_ld, void* dres, int dres_ld, step_stream_t stream) {
  return act_bwd_launch<__half>(dy, dy_ld, y, y_ld, scale, relu, M, C, dz, dz_ld, dres, dres_ld, stream);
}

extern "C" int step_act_bwd_f32(const float* dy, int dy_ld, const float* y, int y_ld, const float* scale, int relu, long long M, int C,
                                float* dz, int dz_ld, float* dres, int dres_ld, step_stream_t stream) {
  return act_bwd_launch<float>(dy, dy_ld, y, y_ld, scale, relu, M, C, dz, dz_ld, dres, dres_ld, stream);
}

template <typename T>
static int colsum_launch(const void* x, int ld, long long M, int C, float scale, float* out, float* workspace, step_stream_t stream) {
  STEP_CHECK_ARG(x && out && workspace && M > 0 && C > 0, "colsum: bad arguments");
  const int chunks = (int)(M < 64 ? M : 64);
  const int rows_per = ceil_div(M, chunks);
  colsum_partial_kernel<T><<<dim3(ceil_div(C, 256), chunks), 256, 0, cu(stream)>>>((const T*)x, ld, M, C, rows_per, workspace);
  STEP_LAUNCH_CHECK("colsum_partial_kernel");
  colsum_reduce_kernel<<<ceil_div(C, 256), 256, 0, cu(stream)>>>(workspace, chunks, C, scale, out);
  STEP_LAUNCH_CHECK("colsum_reduce_kernel");
  return 0;
}

extern "C" int step_colsum_f16(const void* x, int ld, long long M, int C, float scale, float* out, float* workspace /* >= 64*C floats */,
                               step_stream_t stream) {
  return colsum_launch<__half>(x, ld, M, C, scale, out, workspace, stream);
}

extern "C" int step_colsum_f32(const float* x, int ld, long long M, int C, float scale, float* out, float* workspace /* >= 64*C floats */,
                               step_stream_t stream) {
  return colsum_launch<float>(x, ld, M, C, scale, out, workspace, stream);
}

template <typename T>
static int mean_mid_bwd_launch(const float* g, int A, int B, int P, int C, float gscale, void* dx, int ld, step_stream_t stream) {
  STEP_CHECK_ARG(g && dx && A > 0 && B > 0 && P > 0 && C > 0 && ld >= C, "mean_mid_bwd: bad arguments");
  mean_mid_bwd_kernel<T, false><<<ceil_div((long long)A * B * P * C, 256), 256, 0, cu(stream)>>>(g, A, B, P, C, gscale, (T*)dx, ld,
                                                                                                  DropDraw{}, DropMap{});
  STEP_LAUNCH_CHECK("mean_mid_bwd_kernel");
  return 0;
}

extern "C" int step_mean_mid_bwd(const float* g, int A, int B, int P, int C, float gscale, void* dx, int ld, step_stream_t stream) {
  return mean_mid_bwd_launch<__half>(g, A, B, P, C, gscale, dx, ld, stream);
}

extern "C" int step_mean_mid_bwd_f32(const float* g, int A, int B, int P, int C, float gscale, float* dx, int ld, step_stream_t stream) {
  return mean_mid_bwd_launch<float>(g, A, B, P, C, gscale, dx, ld, stream);
}

extern "C" int step_f32_accum_f16(const float* src, long long M, int C, float gscale, void* dst, int ld, step_stream_t stream) {
  STEP_CHECK_ARG(src && dst && M > 0 && C > 0 && ld >= C, "f32_accum_f16: bad arguments");
  f32_accum_f16_kernel<false><<<ceil_div(M * C, 256), 256, 0, cu(stream)>>>(src, M, C, gscale, (__half*)dst, ld, 1, DropDraw{}, DropMap{});
  STEP_LAUNCH_CHECK("f32_accum_f16_kernel");
  return 0;
}

extern "C" int step_f32_accum_f32(const float* src, long long M, int C, float gscale, float* dst, int ld, step_stream_t stream) {
  STEP_CHECK_ARG(src && dst && M > 0 && C > 0 && ld >= C, "f32_accum_f32: bad arguments");
  f32_accum_f32_kernel<false><<<ceil_div(M * C, 256), 256, 0, cu(stream)>>>(src, M, C, gscale, dst, ld, 1, DropDraw{}, DropMap{});
  STEP_LAUNCH_CHECK("f32_accum_f32_kernel");
  return 0;
}

template <typename T>
static int maxpool3d_bwd_launch(const void* x, int x_ld, const void* dy, int dy_ld, int N, int T_, int H, int W, int C, int KT,
                                int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                                int pad_hi_w, int OT, int OH, int OW, void* dx, int dx_ld, uint8_t* argmax_ws, step_stream_t stream) {
  STEP_CHECK_ARG(x && dy && dx && argmax_ws && N > 0 && T_ > 0 && H > 0 && W > 0 && C > 0 && KT * KH * KW < 254, "maxpool3d_bwd: bad arguments");
  // the argmax pass divides by the strides, and a window must start inside its padding for every tap index to fit a byte
  STEP_CHECK_ARG(KT > 0 && KH > 0 && KW > 0 && ST > 0 && SH > 0 && SW > 0 && OT > 0 && OH > 0 && OW > 0,
                 "maxpool3d_bwd: kernel %dx%dx%d, stride %dx%dx%d, output %dx%dx%d must be positive", KT, KH, KW, ST, SH, SW, OT, OH, OW);
  STEP_CHECK_ARG(PT >= 0 && PT < KT && PH >= 0 && PH < KH && PW >= 0 && PW < KW && pad_hi_t >= 0 && pad_hi_h >= 0 && pad_hi_w >= 0,
                 "maxpool3d_bwd: bad padding (%d,%d,%d) / (%d,%d,%d) for kernel %dx%dx%d", PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w, KT, KH, KW);
  PoolGeom g = {N, T_, H, W, C, KT, KH, KW, ST, SH, SW, PT, PH, PW, OT, OH, OW, pad_hi_t, pad_hi_h, pad_hi_w};
  const long long n_out = (long long)N * OT * OH * OW * C, n_in = (long long)N * T_ * H * W * C;
  maxpool_argmax_kernel<T><<<ceil_div(n_out, 256), 256, 0, cu(stream)>>>(g, (const T*)x, x_ld, argmax_ws);
  STEP_LAUNCH_CHECK("maxpool_argmax_kernel");
  maxpool_bwd_kernel<T><<<ceil_div(n_in, 256), 256, 0, cu(stream)>>>(g, (const T*)dy, dy_ld, argmax_ws, (T*)dx, dx_ld);
  STEP_LAUNCH_CHECK("maxpool_bwd_kernel");
  return 0;
}

extern "C" int step_maxpool3d_bwd_f16(const void* x, int x_ld, const void* dy, int dy_ld, int N, int T, int H, int W, int C, int KT,
                                      int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                                      int pad_hi_w, int OT, int OH, int OW, void* dx /* accumulated in place */, int dx_ld, uint8_t* argmax_ws /* N*OT*OH*OW*C bytes */,
                                      step_stream_t stream) {
  return maxpool3d_bwd_launch<__half>(x, x_ld, dy, dy_ld, N, T, H, W, C, KT, KH, KW, ST, SH, SW, PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w,
                                      OT, OH, OW, dx, dx_ld, argmax_ws, stream);
}

extern "C" int step_maxpool3d_bwd_f32(const float* x, int x_ld, const float* dy, int dy_ld, int N, int T, int H, int W, int C, int KT,
                                      int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                                      int pad_hi_w, int OT, int OH, int OW, float* dx /* accumulated in place */, int dx_ld, uint8_t* argmax_ws,
                                      step_stream_t stream) {
  return maxpool3d_bwd_launch<float>(x, x_ld, dy, dy_ld, N, T, H, W, C, KT, KH, KW, ST, SH, SW, PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w,
                                     OT, OH, OW, dx, dx_ld, argmax_ws, stream);
}

extern "C" size_t step_conv_wgrad_f32_workspace_bytes(long long M, int Cout, int Cin, int taps) {
  if (M <= 0 || Cout <= 0 || Cin <= 0 || taps <= 0) return 0;
  const WfPlan p = wgrad_f32_plan(M, Cout, (long long)taps * Cin);
  return (size_t)p.chunks * p.tiles_co * p.tiles_j * kWfTile * kWfTile * sizeof(float);
}

extern "C" int step_conv_wgrad_f32(const float* dz, int dz_ld, const float* x, int x_ld, int N, int T, int H, int W, int OT, int OH,
                                   int OW, int Cout, int Cin, int KT, int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW,
                                   float scale, float* dw, int dw_ld, int accumulate, void* workspace, size_t ws_bytes,
                                   step_stream_t stream) {
  STEP_CHECK_ARG(N > 0 && T > 0 && H > 0 && W > 0 && OT > 0 && OH > 0 && OW > 0 && Cout > 0 && Cin > 0 && KT > 0 && KH > 0 && KW > 0 &&
                 ST > 0 && SH > 0 && SW > 0 && dz && x && dw && workspace, "conv_wgrad_f32: bad arguments");
  const long long M = (long long)N * OT * OH * OW, cols = (long long)KT * KH * KW * Cin;
  STEP_CHECK_ARG(M < (1LL << 31) && (long long)N * T * H * W < (1LL << 31) && cols < (1LL << 31),
                 "conv_wgrad_f32: %lld output pixels / %lld weight columns exceed 2^31", M, cols);
  STEP_CHECK_ARG(Cout % 4 == 0 && Cin % 4 == 0 && dz_ld % 4 == 0 && x_ld % 4 == 0 && dz_ld >= Cout && x_ld >= Cin && dw_ld >= Cin,
                 "conv_wgrad_f32: channel counts / strides must be multiples of 4 (Cout=%d Cin=%d dz_ld=%d x_ld=%d dw_ld=%d)",
                 Cout, Cin, dz_ld, x_ld, dw_ld);
  STEP_CHECK_ARG((((uintptr_t)dz | (uintptr_t)x) & 15) == 0, "conv_wgrad_f32: pointers must be 16-byte aligned");
  STEP_CHECK_ARG(PT >= 0 && PT < KT && PH >= 0 && PH < KH && PW >= 0 && PW < KW, "conv_wgrad_f32: bad padding");
  // every output pixel's first tap lies inside the padded input (as step_conv3d_fwd requires)
  STEP_CHECK_ARG((OT - 1) * ST - PT < T && (OH - 1) * SH - PH < H && (OW - 1) * SW - PW < W,
                 "conv_wgrad_f32: output extent %dx%dx%d inconsistent with input %dx%dx%d / stride / pad", OT, OH, OW, T, H, W);
  const size_t need = step_conv_wgrad_f32_workspace_bytes(M, Cout, Cin, KT * KH * KW);
  if (ws_bytes < need) return fail(STEP_E_WORKSPACE, "conv_wgrad_f32: workspace %zu < %zu", ws_bytes, need);
  const WfPlan p = wgrad_f32_plan(M, Cout, cols);
  STEP_CHECK_ARG(p.tiles_j <= 65535 && p.chunks <= 65535, "conv_wgrad_f32: grid too large");
  const WfGeom g = {T, H, W, OT, OH, OW, KH, KW, ST, SH, SW, PT, PH, PW, Cin, (int)cols, (int)M, p.chunk};
  conv_wgrad_f32_partial_kernel<<<dim3(p.tiles_co, p.tiles_j, p.chunks), 256, 0, cu(stream)>>>(dz, dz_ld, x, x_ld, Cout, g,
                                                                                               (float*)workspace);
  STEP_LAUNCH_CHECK("conv_wgrad_f32_partial_kernel");
  conv_wgrad_f32_reduce_kernel<<<ceil_div((long long)Cout * cols, 256), 256, 0, cu(stream)>>>((const float*)workspace, p.chunks, p.tiles_co,
                                                                                              p.tiles_j, Cout, Cin, (int)cols, scale, dw,
                                                                                              dw_ld, accumulate);
  STEP_LAUNCH_CHECK("conv_wgrad_f32_reduce_kernel");
  return 0;
}

// ---- dropout entries -------------------------------------------------------------------------------------------------------
// torch's launch geometry for a draw of n elements (dropout.cuh); the argument checks every dropout entry makes first
static int make_draw(const step_dropout_draw* d, long long n, const char* who, DropDraw* out, unsigned long long* offset_step) {
  STEP_CHECK_ARG(d, "%s: null draw", who);
  STEP_CHECK_ARG(d->keep > 0.0f && d->keep < 1.0f, "%s: keep probability %g outside (0, 1) (torch draws nothing at p = 0 or 1)", who,
                 (double)d->keep);
  STEP_CHECK_ARG(d->sm_count > 0 && d->threads_per_sm >= 256, "%s: sm_count %d / threads_per_sm %d must be positive and >= 256", who,
                 d->sm_count, d->threads_per_sm);
  if (n <= 0 || n % 4 != 0 || n > 0x7fffffffLL)
    return fail(STEP_E_UNSUPPORTED, "%s: a draw of %lld elements (only 0 < n < 2^31 with n %% 4 == 0 is reproduced)", who, n);
  const long long grid = std::min((n + 255) / 256, (long long)d->sm_count * (d->threads_per_sm / 256));
  if (out) *out = DropDraw{(unsigned long long)d->seed, (unsigned long long)d->offset, d->keep, (float)(1.0 / (double)d->keep),
                           (unsigned int)(grid * 256)};
  if (offset_step) *offset_step = (unsigned long long)(((n - 1) / (grid * 256 * 4) + 1) * 4);
  return 0;
}

// the global draw's tensor [R, C' = C*P + ctx_cols, T_len] (two_branch.py:239-244): element (r, t, p, c) of the downsample
// output is (r * C' + c * P + p) * T_len + t; with base C*P*T_len and channel stride T_len, (r, t, 0, k) is context column k
static DropMap global_map(int T_len, int P, int C, int ctx_cols, bool context) {
  const long long Cp = (long long)C * P + ctx_cols;
  if (context) return DropMap{(long long)C * P * T_len, Cp * T_len, 1, 0, T_len};
  return DropMap{0, Cp * T_len, 1, T_len, P * T_len};
}
// the local draw's tensor [F, C, P] (two_branch.py:259-261): element (f, 0, p, c) is (f * C + c) * P + p
static DropMap local_map(int P, int C) { return DropMap{0, (long long)C * P, 0, 1, P}; }

extern "C" int step_dropout_check(const step_dropout_draw* draw, long long n, uint64_t* offset_step) {
  unsigned long long s = 0;
  if (int rc = make_draw(draw, n, "dropout", nullptr, &s)) return rc;
  if (offset_step) *offset_step = s;
  return 0;
}

extern "C" int step_dropout_mask_u8(const step_dropout_draw* draw, long long n, uint8_t* mask, step_stream_t stream) {
  DropDraw dd;
  if (int rc = make_draw(draw, n, "dropout_mask_u8", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(mask, "dropout_mask_u8: null pointer");
  dropout_mask_kernel<<<(unsigned)std::min((n + 255) / 256, 8LL * kNumSMs * 8), 256, 0, cu(stream)>>>(dd, n, mask);
  STEP_LAUNCH_CHECK("dropout_mask_kernel");
  return 0;
}

template <typename T>
static int dropout_copy_launch(const DropDraw& dd, const DropMap& mp, const void* x, int x_ld, long long M, int T_len, int P, int C,
                               void* y, int y_ld, step_stream_t stream) {
  dropout_copy_kernel<T><<<ceil_div(M * C, 256), 256, 0, cu(stream)>>>((const T*)x, x_ld, M, T_len, P, C, (T*)y, y_ld, dd, mp);
  STEP_LAUNCH_CHECK("dropout_copy_kernel");
  return 0;
}

extern "C" int step_dropout_global_fwd(const step_dropout_draw* draw, const void* x, int dtype, int x_ld, int R, int T_len, int P,
                                       int C, int ctx_cols, void* y, int y_ld, step_stream_t stream) {
  STEP_CHECK_ARG(R > 0 && T_len > 0 && P > 0 && C > 0 && ctx_cols >= 0 && x_ld >= C && y_ld >= C,
                 "dropout_global_fwd: bad shape R=%d T=%d P=%d C=%d ctx_cols=%d x_ld=%d y_ld=%d", R, T_len, P, C, ctx_cols, x_ld, y_ld);
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)R * ((long long)C * P + ctx_cols) * T_len, "dropout_global_fwd", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(x && y, "dropout_global_fwd: null pointer");
  const DropMap mp = global_map(T_len, P, C, ctx_cols, false);
  const long long M = (long long)R * T_len * P;
  if (dtype == STEP_F32) return dropout_copy_launch<float>(dd, mp, x, x_ld, M, T_len, P, C, y, y_ld, stream);
  if (dtype == STEP_F16) return dropout_copy_launch<__half>(dd, mp, x, x_ld, M, T_len, P, C, y, y_ld, stream);
  return fail(STEP_E_ARG, "dropout_global_fwd: dtype %d", dtype);
}

extern "C" int step_dropout_local_fwd(const step_dropout_draw* draw, const void* x, int dtype, int x_ld, int F, int P, int C, void* y,
                                      int y_ld, step_stream_t stream) {
  STEP_CHECK_ARG(F > 0 && P > 0 && C > 0 && x_ld >= C && y_ld >= C, "dropout_local_fwd: bad shape F=%d P=%d C=%d x_ld=%d y_ld=%d", F, P,
                 C, x_ld, y_ld);
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)F * C * P, "dropout_local_fwd", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(x && y, "dropout_local_fwd: null pointer");
  const DropMap mp = local_map(P, C);
  const long long M = (long long)F * P;
  if (dtype == STEP_F32) return dropout_copy_launch<float>(dd, mp, x, x_ld, M, 1, P, C, y, y_ld, stream);
  if (dtype == STEP_F16) return dropout_copy_launch<__half>(dd, mp, x, x_ld, M, 1, P, C, y, y_ld, stream);
  return fail(STEP_E_ARG, "dropout_local_fwd: dtype %d", dtype);
}

extern "C" int step_dropout_ctx_mean_f32(const step_dropout_draw* draw, int P, int C, const float* ctx, const int32_t* row_map,
                                         long long row_stride, int t_stride, int k_stride, int R, int T_len, int K, float* out,
                                         step_stream_t stream) {
  STEP_CHECK_ARG(R > 0 && T_len > 0 && K > 0 && P > 0 && C > 0 && row_stride >= 0 && t_stride >= 0 && k_stride >= 0,
                 "dropout_ctx_mean_f32: bad shape R=%d T=%d K=%d P=%d C=%d", R, T_len, K, P, C);
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)R * ((long long)C * P + K) * T_len, "dropout_ctx_mean_f32", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(ctx && out, "dropout_ctx_mean_f32: null pointer");
  ctx_mean_dropout_kernel<<<ceil_div((long long)R * K, 256), 256, 0, cu(stream)>>>(ctx, row_map, row_stride, t_stride, k_stride, R, T_len,
                                                                                   K, out, dd, global_map(T_len, P, C, K, true));
  STEP_LAUNCH_CHECK("ctx_mean_dropout_kernel");
  return 0;
}

extern "C" int step_mean_mid_bwd_dropout(const step_dropout_draw* draw, int ctx_cols, const float* g, int A, int B, int P, int C,
                                         float gscale, void* dx, int dtype, int ld, step_stream_t stream) {
  STEP_CHECK_ARG(A > 0 && B > 0 && P > 0 && C > 0 && ctx_cols >= 0 && ld >= C, "mean_mid_bwd_dropout: bad arguments");
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)A * ((long long)C * P + ctx_cols) * B, "mean_mid_bwd_dropout", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(g && dx, "mean_mid_bwd_dropout: null pointer");
  const DropMap mp = global_map(B, P, C, ctx_cols, false);
  const int grid = ceil_div((long long)A * B * P * C, 256);
  if (dtype == STEP_F32)
    mean_mid_bwd_kernel<float, true><<<grid, 256, 0, cu(stream)>>>(g, A, B, P, C, gscale, (float*)dx, ld, dd, mp);
  else if (dtype == STEP_F16)
    mean_mid_bwd_kernel<__half, true><<<grid, 256, 0, cu(stream)>>>(g, A, B, P, C, gscale, (__half*)dx, ld, dd, mp);
  else
    return fail(STEP_E_ARG, "mean_mid_bwd_dropout: dtype %d", dtype);
  STEP_LAUNCH_CHECK("mean_mid_bwd_kernel");
  return 0;
}

extern "C" int step_f32_accum_dropout(const step_dropout_draw* draw, const float* src, int F, int P, int C, float gscale, void* dst,
                                      int dtype, int ld, step_stream_t stream) {
  STEP_CHECK_ARG(F > 0 && P > 0 && C > 0 && ld >= C, "f32_accum_dropout: bad arguments");
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)F * C * P, "f32_accum_dropout", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(src && dst, "f32_accum_dropout: null pointer");
  const long long M = (long long)F * P;
  const DropMap mp = local_map(P, C);
  if (dtype == STEP_F32)
    f32_accum_f32_kernel<true><<<ceil_div(M * C, 256), 256, 0, cu(stream)>>>(src, M, C, gscale, (float*)dst, ld, P, dd, mp);
  else if (dtype == STEP_F16)
    f32_accum_f16_kernel<true><<<ceil_div(M * C, 256), 256, 0, cu(stream)>>>(src, M, C, gscale, (__half*)dst, ld, P, dd, mp);
  else
    return fail(STEP_E_ARG, "f32_accum_dropout: dtype %d", dtype);
  STEP_LAUNCH_CHECK("f32_accum_dropout_kernel");
  return 0;
}

extern "C" int step_ctx_grad_reduce_dropout_f32(const step_dropout_draw* draw, int P, int Cg, const float* dctx, int dctx_ld,
                                                const float* tubes, int R, int T_len, int B, int feat_T, int t_start, int C, float* acc,
                                                step_stream_t stream) {
  STEP_CHECK_ARG(B > 0 && C > 0 && R > 0 && T_len > 0 && P > 0 && Cg > 0 && dctx_ld >= C && t_start >= 0 && t_start + T_len <= feat_T,
                 "ctx_grad_reduce_dropout: bad shape B=%d C=%d R=%d T_len=%d feat_T=%d t_start=%d", B, C, R, T_len, feat_T, t_start);
  DropDraw dd;
  if (int rc = make_draw(draw, (long long)R * ((long long)Cg * P + C) * T_len, "ctx_grad_reduce_dropout", &dd, nullptr)) return rc;
  STEP_CHECK_ARG(acc && dctx && tubes, "ctx_grad_reduce_dropout: null pointer");
  ctx_grad_reduce_kernel<true><<<ceil_div((long long)B * C, 256), 256, 0, cu(stream)>>>(dctx, dctx_ld, tubes, R, T_len, B, feat_T, t_start,
                                                                                        C, acc, dd, global_map(T_len, P, Cg, C, true));
  STEP_LAUNCH_CHECK("ctx_grad_reduce_kernel");
  return 0;
}

