// roi.cu -- ROIAlign / ROIPool for sm_90a.
//
// Replaces _C.roi_align_forward/backward and _C.roi_pool_forward/backward
// (external/maskrcnn_benchmark/csrc/vision.cpp:32-35).  Arithmetic follows
// cpu/ROIAlign_cpu.cpp:41-243 == cuda/ROIAlign_cuda.cu:39-146 and cuda/ROIPool_cuda.cu:40-132:
// legacy (aligned=False) sampling, roi extent forced to >= 1, adaptive grid ceil(roi/pooled) when
// sampling_ratio == 0, samples outside [-1, H] contribute 0, 4-tap bilinear, mean over the grid.
// Every fp32 operation is explicitly rounded (__fmul_rn / __fadd_rn / __fdiv_rn, no FMA
// contraction) in the reference's operand order, so the fp32 kernels are bit-identical to the
// reference CPU op.
//
// Two data layouts:
//   *_nchw_f32 : the reference's own layout, one thread per output element (compat boundary).
//   *_nhwc     : channels-last fast path used inside the pipeline.  One CTA per ROI row builds the
//                tap table (<= 49 bins x gh x gw samples) once in shared memory, then every thread
//                streams 16-byte channel vectors: loads and stores are fully coalesced along C,
//                tap weights are shared by all channels, the feature map stays L2 resident
//                (42 MB at C4 vs 126 MB L2) and HBM traffic is the compulsory output write.
// The layouts above are the forwards'.  The backwards of both layouts have no atomics and share one kernel body per
// operation, parameterised by strides ("Backward, both layouts" below).
#include "roi_math.cuh"

namespace step {

// ------------------------------------------------------------------------------------------
// NCHW fp32 (reference layout)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) roi_align_fwd_nchw_kernel(long long total, const float* __restrict__ feat,
                                                                 float scale, int C, int H, int W, int ph,
                                                                 int pw, int sampling_ratio,
                                                                 const float* __restrict__ rois,
                                                                 float* __restrict__ out) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int q = (int)(idx % pw);
    int p = (int)((idx / pw) % ph);
    int c = (int)((idx / pw / ph) % C);
    int n = (int)(idx / pw / ph / C);
    RoiGeom g = roi_geometry(rois + 5 * (size_t)n, scale, ph, pw, sampling_ratio);
    const float* plane = feat + ((size_t)g.batch * C + c) * H * W;
    float acc = 0.0f;
    for (int iy = 0; iy < g.gh; ++iy) {
      float y = sample_coord(g.start_h, p, g.bin_h, iy, g.gh);
      for (int ix = 0; ix < g.gw; ++ix) {
        float x = sample_coord(g.start_w, q, g.bin_w, ix, g.gw);
        Tap t = make_tap(H, W, y, x);
        if (t.p1 >= 0)
          acc = __fadd_rn(acc, tap_dot(t, __ldg(plane + t.p1), __ldg(plane + t.p2), __ldg(plane + t.p3),
                                       __ldg(plane + t.p4)));
      }
    }
    out[idx] = __fdiv_rn(acc, g.count);
  }
}

struct PoolWin { int batch, hs, he, ws, we; };

__device__ __forceinline__ PoolWin pool_window(const float* __restrict__ roi, float scale, int ph, int pw,
                                               int p, int q, int H, int W) {
  // ROIPool_cuda.cu:51-77
  PoolWin o;
  o.batch = (int)roi[0];
  int sw = (int)roundf(__fmul_rn(roi[1], scale)), sh = (int)roundf(__fmul_rn(roi[2], scale));
  int ew = (int)roundf(__fmul_rn(roi[3], scale)), eh = (int)roundf(__fmul_rn(roi[4], scale));
  int rw = max(ew - sw + 1, 1), rh = max(eh - sh + 1, 1);
  float bin_h = __fdiv_rn((float)rh, (float)ph), bin_w = __fdiv_rn((float)rw, (float)pw);
  int hs = (int)floorf(__fmul_rn((float)p, bin_h)), ws = (int)floorf(__fmul_rn((float)q, bin_w));
  int he = (int)ceilf(__fmul_rn((float)(p + 1), bin_h)), we = (int)ceilf(__fmul_rn((float)(q + 1), bin_w));
  o.hs = min(max(hs + sh, 0), H); o.he = min(max(he + sh, 0), H);
  o.ws = min(max(ws + sw, 0), W); o.we = min(max(we + sw, 0), W);
  return o;
}

__global__ void __launch_bounds__(256) roi_pool_fwd_nchw_kernel(long long total, const float* __restrict__ feat,
                                                                float scale, int C, int H, int W, int ph,
                                                                int pw, const float* __restrict__ rois,
                                                                float* __restrict__ out,
                                                                int32_t* __restrict__ argmax) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int q = (int)(idx % pw);
    int p = (int)((idx / pw) % ph);
    int c = (int)((idx / pw / ph) % C);
    int n = (int)(idx / pw / ph / C);
    PoolWin o = pool_window(rois + 5 * (size_t)n, scale, ph, pw, p, q, H, W);
    bool empty = (o.he <= o.hs) || (o.we <= o.ws);
    float maxval = empty ? 0.0f : -3.402823466e+38f;
    int maxidx = -1;
    const float* plane = feat + ((size_t)o.batch * C + c) * H * W;
    for (int h = o.hs; h < o.he; ++h)
      for (int w = o.ws; w < o.we; ++w) {
        float v = __ldg(plane + h * W + w);
        if (v > maxval) { maxval = v; maxidx = h * W + w; }
      }
    out[idx] = maxval;
    argmax[idx] = maxidx;
  }
}

// ------------------------------------------------------------------------------------------
// NHWC fast path
// ------------------------------------------------------------------------------------------
// ROI column 0 is a frame index into the *sliced* feature map conv_feat[:, t0:t0+roi_T]
// (utils.py:48, tube_utils.py:238).  The pipeline keeps the full [B, feat_T, H, W, C] map and
// remaps instead of materialising the slice.
struct FrameMap {
  int roi_T, feat_T, t0;
  __device__ __forceinline__ int map(int f) const {
    return roi_T > 0 ? (f / roi_T) * feat_T + t0 + (f % roi_T) : f;
  }
};

// kExact: the reference's operation order with explicitly rounded fp32 ops (bit-identical results).
// !kExact (fp16 storage only): the 1/count factor is folded into the tap weights and each tap is one FFMA
// (fp32 accumulate): 1/3 fewer instructions on an issue-bound kernel; results differ from the exact path by
// at most one fp16 ulp after the final rounding (convex combination, no cancellation).
template <typename T, bool kExact>
__global__ void __launch_bounds__(256) roi_align_fwd_nhwc_kernel(const T* __restrict__ feat, int H, int W, int C,
                                                                 int feat_ld, const float* __restrict__ rois,
                                                                 float scale, int ph, int pw, int sampling_ratio,
                                                                 T* __restrict__ out, int out_ld, FrameMap fm) {
  constexpr int VN = Vec16<T>::N;
  __shared__ Tap taps[kMaxTaps];
  const int r = blockIdx.x;
  const RoiGeom g = roi_geometry(rois + 5 * (size_t)r, scale, ph, pw, sampling_ratio);
  const int spb = g.gh * g.gw;  // samples per bin
  const int nbins = ph * pw;
  const bool cached = nbins * spb <= kMaxTaps;
  if (cached) {
    for (int i = threadIdx.x; i < nbins * spb; i += blockDim.x) {
      int bin = i / spb, s = i - bin * spb;
      int p = bin / pw, q = bin - p * pw;
      int iy = s / g.gw, ix = s - iy * g.gw;
      Tap t = make_tap(H, W, sample_coord(g.start_h, p, g.bin_h, iy, g.gh),
                       sample_coord(g.start_w, q, g.bin_w, ix, g.gw));
      if (!kExact) { const float ic = 1.0f / g.count; t.w1 *= ic; t.w2 *= ic; t.w3 *= ic; t.w4 *= ic; }
      taps[i] = t;
    }
    __syncthreads();
  }
  const T* fbase = feat + (size_t)fm.map(g.batch) * H * W * feat_ld;
  T* obase = out + (size_t)r * nbins * out_ld;
  const int nvec = C / VN;
  // count is a power of two in the common case (grid 1x1, 1x2, 2x2): x / 2^k == x * 2^-k exactly
  const bool pow2 = (spb & (spb - 1)) == 0;
  const float inv = 1.0f / g.count;
  for (int item = threadIdx.x; item < nbins * nvec; item += blockDim.x) {
    const int bin = item / nvec, cv = item - bin * nvec;
    float acc[VN];
#pragma unroll
    for (int k = 0; k < VN; ++k) acc[k] = 0.0f;
    for (int s = 0; s < spb; ++s) {
      Tap t;
      if (cached) {
        t = taps[bin * spb + s];
      } else {
        int p = bin / pw, q = bin - p * pw;
        int iy = s / g.gw, ix = s - iy * g.gw;
        t = make_tap(H, W, sample_coord(g.start_h, p, g.bin_h, iy, g.gh),
                     sample_coord(g.start_w, q, g.bin_w, ix, g.gw));
        if (!kExact) { const float ic = 1.0f / g.count; t.w1 *= ic; t.w2 *= ic; t.w3 *= ic; t.w4 *= ic; }
      }
      if (t.p1 < 0) continue;
      float v1[VN], v2[VN], v3[VN], v4[VN];
      load16(fbase + (size_t)t.p1 * feat_ld + cv * VN, v1);
      load16(fbase + (size_t)t.p2 * feat_ld + cv * VN, v2);
      load16(fbase + (size_t)t.p3 * feat_ld + cv * VN, v3);
      load16(fbase + (size_t)t.p4 * feat_ld + cv * VN, v4);
      if (kExact) {
#pragma unroll
        for (int k = 0; k < VN; ++k) acc[k] = __fadd_rn(acc[k], tap_dot(t, v1[k], v2[k], v3[k], v4[k]));
      } else {
#pragma unroll
        for (int k = 0; k < VN; ++k)
          acc[k] = __fmaf_rn(t.w4, v4[k], __fmaf_rn(t.w3, v3[k], __fmaf_rn(t.w2, v2[k], __fmaf_rn(t.w1, v1[k], acc[k]))));
      }
    }
    if (kExact) {
#pragma unroll
      for (int k = 0; k < VN; ++k) acc[k] = pow2 ? __fmul_rn(acc[k], inv) : __fdiv_rn(acc[k], g.count);
    }
    store16(obase + (size_t)bin * out_ld + cv * VN, acc);
  }
}


// fp16 "packed" fast path.  Two observations from profiling the C3 shape: the direct form is bound by
// instruction issue and by the L1 data path (4 taps x g^2 samples = ~10 sixteen-byte loads per 16-byte output).
//  (1) the g^2 samples of a bin hit only <= (g+1)^2 distinct pixels: their bilinear weights are merged per
//      pixel (in fp32, with the 1/count factor) when the per-ROI table is built -> ~5.5 instead of ~10 loads;
//  (2) the weighted sum runs in packed half2 FMAs (the result is a convex combination of the inputs: no
//      cancellation, error <= a few fp16 ulps, far inside the fp16-path tolerance of DESIGN.md section 4).
// ROIs whose bins can touch more than kMaxMerged distinct pixels take a direct form with fp32 FMAs instead.
constexpr int kMaxMerged = 16;
struct MergedBin {
  int n;
  int pad;
  uint2 e[kMaxMerged];   // .x = element offset of the pixel row (pixel index * feat_ld), .y = merged weight as half2 bits
};

__device__ __forceinline__ void hfma2x4(__half2* a, __half2 w, const uint4& v) {
  a[0] = __hfma2(w, *reinterpret_cast<const __half2*>(&v.x), a[0]);
  a[1] = __hfma2(w, *reinterpret_cast<const __half2*>(&v.y), a[1]);
  a[2] = __hfma2(w, *reinterpret_cast<const __half2*>(&v.z), a[2]);
  a[3] = __hfma2(w, *reinterpret_cast<const __half2*>(&v.w), a[3]);
}

template <int V>
__device__ __forceinline__ void roi_gather_items(const MergedBin* bins, int nbins, int nvec, const __half* fbase, __half* obase,
                                                 int out_ld) {
  const int hv = nvec / V;
  int bin = threadIdx.x / hv, cv = threadIdx.x - bin * hv;   // incremental (bin, cv): no per-item division
  const int dbin = blockDim.x / hv, dcv = blockDim.x - dbin * hv;
  const __half2 z2 = __float2half2_rn(0.0f);
  while (bin < nbins) {
    const MergedBin& b = bins[bin];
    __half2 acc[V][4];
#pragma unroll
    for (int u = 0; u < V; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = z2;
    const __half* fp = fbase + cv * 8;
    const int n = b.n;
    int e = 0;
    for (; e + 1 < n; e += 2) {
      const uint2 e0 = b.e[e], e1 = b.e[e + 1];          // one 8-byte shared load per entry
      const __half2 w0 = *reinterpret_cast<const __half2*>(&e0.y), w1 = *reinterpret_cast<const __half2*>(&e1.y);
      uint4 v0[V], v1[V];
#pragma unroll
      for (int u = 0; u < V; ++u) {
        v0[u] = *reinterpret_cast<const uint4*>(fp + e0.x + u * hv * 8);
        v1[u] = *reinterpret_cast<const uint4*>(fp + e1.x + u * hv * 8);
      }
#pragma unroll
      for (int u = 0; u < V; ++u) { hfma2x4(acc[u], w0, v0[u]); hfma2x4(acc[u], w1, v1[u]); }
    }
    if (e < n) {
      const uint2 e0 = b.e[e];
      const __half2 w0 = *reinterpret_cast<const __half2*>(&e0.y);
#pragma unroll
      for (int u = 0; u < V; ++u) hfma2x4(acc[u], w0, *reinterpret_cast<const uint4*>(fp + e0.x + u * hv * 8));
    }
    __half* op = obase + (size_t)bin * out_ld + cv * 8;
#pragma unroll
    for (int u = 0; u < V; ++u) *reinterpret_cast<uint4*>(op + u * hv * 8) = *reinterpret_cast<const uint4*>(acc[u]);
    bin += dbin; cv += dcv;
    if (cv >= hv) { cv -= hv; ++bin; }
  }
}


// 5 CTAs of 256 threads per SM: at most 51 registers (48 in use; without the bound the compiler takes 59).
__global__ void __launch_bounds__(256, 5) roi_align_fwd_nhwc_f16_packed_kernel(const __half* __restrict__ feat, int H, int W,
                                                                            int C, int feat_ld, const float* __restrict__ rois,
                                                                            float scale, int ph, int pw, int sampling_ratio,
                                                                            __half* __restrict__ out, int out_ld, FrameMap fm) {
  extern __shared__ MergedBin bins[];  // [ph * pw]
  const int r = blockIdx.x;
  const RoiGeom g = roi_geometry(rois + 5 * (size_t)r, scale, ph, pw, sampling_ratio);
  const int nbins = ph * pw;
  const __half* fbase = feat + (size_t)fm.map(g.batch) * H * W * feat_ld;
  const int nvec = C >> 3;
  // Distinct pixels one bin can touch, per axis: g + 1 when its g samples are at most one pixel apart (the bin is no wider
  // than g pixels, always so for the adaptive grid), else two per sample.
  const int nh = g.bin_h <= (float)g.gh ? g.gh + 1 : 2 * g.gh, nw = g.bin_w <= (float)g.gw ? g.gw + 1 : 2 * g.gw;
  if (nh * nw > kMaxMerged) {
    // a bin may not fit the table (sampling grid > 3x3, or a fixed sampling_ratio with bins wider than the grid):
    // direct form with fp32 FMAs, no table
    const float ic = 1.0f / g.count;
    __half* obase = out + (size_t)r * nbins * out_ld;
    for (int item = threadIdx.x; item < nbins * nvec; item += blockDim.x) {
      const int bin = item / nvec, cv = item - bin * nvec;
      const int p = bin / pw, q = bin - p * pw;
      float acc[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
      for (int iy = 0; iy < g.gh; ++iy)
        for (int ix = 0; ix < g.gw; ++ix) {
          Tap t = make_tap(H, W, sample_coord(g.start_h, p, g.bin_h, iy, g.gh), sample_coord(g.start_w, q, g.bin_w, ix, g.gw));
          if (t.p1 < 0) continue;
          float v1[8], v2[8], v3[8], v4[8];
          load16(fbase + (size_t)t.p1 * feat_ld + cv * 8, v1);
          load16(fbase + (size_t)t.p2 * feat_ld + cv * 8, v2);
          load16(fbase + (size_t)t.p3 * feat_ld + cv * 8, v3);
          load16(fbase + (size_t)t.p4 * feat_ld + cv * 8, v4);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            acc[k] = fmaf(t.w4 * ic, v4[k], fmaf(t.w3 * ic, v3[k], fmaf(t.w2 * ic, v2[k], fmaf(t.w1 * ic, v1[k], acc[k]))));
        }
      store16(obase + (size_t)bin * out_ld + cv * 8, acc);
    }
    return;
  }
  for (int bin = threadIdx.x; bin < nbins; bin += blockDim.x) {
    const int p = bin / pw, q = bin - p * pw;
    const float ic = 1.0f / g.count;
    int n = 0;
    int pos[kMaxMerged];
    float wt[kMaxMerged];
    for (int iy = 0; iy < g.gh; ++iy)
      for (int ix = 0; ix < g.gw; ++ix) {
        Tap t = make_tap(H, W, sample_coord(g.start_h, p, g.bin_h, iy, g.gh), sample_coord(g.start_w, q, g.bin_w, ix, g.gw));
        if (t.p1 < 0) continue;
        const int tp[4] = {t.p1, t.p2, t.p3, t.p4};
        const float tw[4] = {t.w1 * ic, t.w2 * ic, t.w3 * ic, t.w4 * ic};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          int e = 0;
          while (e < n && pos[e] != tp[k]) ++e;
          if (e == n) {
            if (n < kMaxMerged) { pos[n] = tp[k]; wt[n] = tw[k]; ++n; }   // n <= nh * nw <= kMaxMerged (above)
          } else {
            wt[e] += tw[k];
          }
        }
      }
    MergedBin& b = bins[bin];
    b.n = n;
    for (int e = 0; e < n; ++e) {
      const __half2 w2 = __float2half2_rn(wt[e]);
      b.e[e] = make_uint2((unsigned)(pos[e] * feat_ld), *reinterpret_cast<const unsigned*>(&w2));
    }
  }
  __syncthreads();
  // Gather: an item is (bin, V channel vectors a V-th of a row apart): the 8-byte table entry (pixel offset, merged
  // weight) is read once for V 16-byte vectors, and two entries are in flight per iteration (2V independent loads).
  // formed here, not before the table build: held across it, obase spills under the 51-register bound
  __half* obase = out + (size_t)r * nbins * out_ld;
  if ((nvec & 1) == 0) roi_gather_items<2>(bins, nbins, nvec, fbase, obase, out_ld);
  else roi_gather_items<1>(bins, nbins, nvec, fbase, obase, out_ld);
}

// kArgmax (training): also record, per output element, the frame-local pixel h*W + w of the maximum in `argmax`
// [R, ph, pw, C] (channel stride C), -1 for an empty bin.  The rule of ROIPool_cuda.cu:79-96: strict `>` against the running
// maximum, h outer / w inner, so on ties the first pixel in scan order wins.  The pooled value is the same fmaxf chain as
// without the flag (`v > m` and fmaxf agree on which value is largest; only the index is added), so outputs are bit-identical.
template <typename T, bool kArgmax>
__global__ void __launch_bounds__(256) roi_pool_fwd_nhwc_kernel(const T* __restrict__ feat, int H, int W, int C,
                                                                int feat_ld, const float* __restrict__ rois,
                                                                float scale, int ph, int pw, T* __restrict__ out,
                                                                int out_ld, FrameMap fm, int32_t* __restrict__ argmax) {
  constexpr int VN = Vec16<T>::N;
  const int r = blockIdx.x, nbins = ph * pw, nvec = C / VN;
  T* obase = out + (size_t)r * nbins * out_ld;
  for (int item = threadIdx.x; item < nbins * nvec; item += blockDim.x) {
    const int bin = item / nvec, cv = item - bin * nvec;
    const int p = bin / pw, q = bin - p * pw;
    PoolWin o = pool_window(rois + 5 * (size_t)r, scale, ph, pw, p, q, H, W);
    const bool empty = (o.he <= o.hs) || (o.we <= o.ws);
    float m[VN];
    int idx[kArgmax ? VN : 1];
#pragma unroll
    for (int k = 0; k < VN; ++k) m[k] = empty ? 0.0f : -3.402823466e+38f;
    if constexpr (kArgmax) {
#pragma unroll
      for (int k = 0; k < VN; ++k) idx[k] = -1;
    }
    const T* fbase = feat + (size_t)fm.map(o.batch) * H * W * feat_ld + cv * VN;
    for (int h = o.hs; h < o.he; ++h)
      for (int w = o.ws; w < o.we; ++w) {
        float v[VN];
        load16(fbase + (size_t)(h * W + w) * feat_ld, v);
        if constexpr (kArgmax) {
#pragma unroll
          for (int k = 0; k < VN; ++k) idx[k] = v[k] > m[k] ? h * W + w : idx[k];
        }
#pragma unroll
        for (int k = 0; k < VN; ++k) m[k] = fmaxf(m[k], v[k]);
      }
    store16(obase + (size_t)bin * out_ld + cv * VN, m);
    if constexpr (kArgmax) {
      int4* a = reinterpret_cast<int4*>(argmax + ((size_t)r * nbins + bin) * C + cv * VN);
#pragma unroll
      for (int k = 0; k < VN / 4; ++k) a[k] = make_int4(idx[4 * k], idx[4 * k + 1], idx[4 * k + 2], idx[4 * k + 3]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Backward, both layouts, no atomics
// ------------------------------------------------------------------------------------------
// The reference scatters both backwards with float atomic adds (ROIAlign_cuda.cu:201-278, ROIPool_cuda.cu:103-132), so its
// sums come out in a different order on every run.  Here a CTA owns a (frame, channel chunk, pixel band) tile of the
// gradient in shared memory, walks the frame's ROI rows in ascending order and adds each row's contribution in a fixed
// order, so every element of grad_in is the same sum, in the same order, whatever the launch geometry:
//   ROIAlign: running sum from +0.0f; per row r of the frame (ascending), the row's samples in (bin, iy, ix) order are
//             taken in slices of kMaxTaps, and per slice that touches the element a partial from +0.0f adds
//             fl(fl(g * w) / count) over the slice's samples, taps p1..p4 in order; the partial is added to the running
//             sum.  (A row of at most kMaxTaps samples -- sampling grids up to 4x4 -- is one slice.)
//   ROIPool:  running sum from +0.0f adds grad_out in ascending (row, ph, pw) order where argmax selects the element.
// What the CTA does with the running sums is its mode: kStore writes them to grad_in frame f (all of [0, K) is written),
// kAdd adds them to frame fm.map(f) (frames without a row get +0.0f), kAddIfRows only for frames with a row.  Rows whose
// frame is outside the launched range belong to no CTA and are ignored.
enum RoiBwdMode { kStore = 0, kAdd = 1, kAddIfRows = 2 };

// Operands of one backward launch.  Strides in elements: grad_out [R, ph, pw, C] (channel stride out_ld) or [R, C, ph, pw];
// argmax (ROIPool) [R, ph, pw, C] or [R, C, ph, pw]; grad_in [K, H, W, C] (channel stride in_ld) or [K, C, H, W].
struct RoiBwdArgs {
  const float* rois;
  int R, ph, pw, sr, H, W, C;
  float scale;
  bool cl;                         // channels-last
  long long go_row, am_row, gi_frame;
  int go_bin, go_c, am_bin, am_c, gi_pix, gi_c;
  const int32_t* argmax;
  float* grad_in;
  FrameMap fm;
  int mode;
  int band_h, band_w;              // ROIAlign: the CTA's pixel tile; ROIPool: band_h pixels (linear), band_w = 1
  int staged;                      // ROIAlign: the row's grad_out chunk is staged in shared memory
};

static RoiBwdArgs roi_bwd_args(bool cl, const float* rois, int R, float scale, int ph, int pw, int sr, int H, int W, int C,
                               int out_ld, int in_ld, const int32_t* argmax, float* grad_in, FrameMap fm, int mode) {
  RoiBwdArgs a{};
  const long long nbins = (long long)ph * pw, npix = (long long)H * W;
  a.rois = rois; a.R = R; a.ph = ph; a.pw = pw; a.sr = sr; a.H = H; a.W = W; a.C = C; a.scale = scale; a.cl = cl;
  a.argmax = argmax; a.grad_in = grad_in; a.fm = fm; a.mode = mode;
  if (cl) {
    a.go_row = nbins * out_ld; a.go_bin = out_ld; a.go_c = 1;
    a.am_row = nbins * C; a.am_bin = C; a.am_c = 1;
    a.gi_frame = npix * in_ld; a.gi_pix = in_ld; a.gi_c = 1;
  } else {
    a.go_row = a.am_row = C * nbins; a.go_bin = a.am_bin = 1; a.go_c = a.am_c = (int)nbins;
    a.gi_frame = C * npix; a.gi_pix = 1; a.gi_c = (int)npix;
  }
  return a;
}

// The ROI rows of frame f, in ascending order, compacted blockDim.x at a time into rows[]: calls body(row) for each with the
// whole CTA.  Returns how many there were.
template <typename Body>
__device__ __forceinline__ int for_each_frame_row(const float* __restrict__ rois, int R, int f, int* rows, int* warp_rows,
                                                  Body body) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = (blockDim.x + 31) >> 5;
  const unsigned mask = blockDim.x >= 32 ? 0xffffffffu : (1u << blockDim.x) - 1u;
  int seen = 0;
  for (int base = 0; base < R; base += blockDim.x) {
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
    for (int j = 0; j < n; ++j) body(rows[j]);
    seen += n;
  }
  return seen;
}

// Hands the CTA's running sums acc (pixel p of the band at acc[p * lda + k] for channel c0 + k) to grad_in by the mode.
__device__ __forceinline__ void roi_bwd_store(const RoiBwdArgs& a, const float* acc, int lda, int f, int c0, int nch, int y0,
                                              int x0, int bh, int bw) {
  float* dst = a.grad_in + (long long)a.fm.map(f) * a.gi_frame;
  const int npx = bh * bw;
  for (int i = threadIdx.x; i < npx * nch; i += blockDim.x) {
    // channel fastest when channels are contiguous, pixel fastest otherwise: coalesced either way
    const int k = a.cl ? i % nch : i / npx, p = a.cl ? i / nch : i % npx;
    const int c = c0 + k;
    if (c >= a.C) continue;
    const int y = y0 + p / bw, x = x0 + p % bw;
    float* d = dst + (long long)(y * a.W + x) * a.gi_pix + (long long)c * a.gi_c;
    const float v = acc[p * lda + k];
    *d = a.mode == kStore ? v : __fadd_rn(*d, v);
  }
}

// ---- ROIAlign -----------------------------------------------------------------------------------------------------------
// CTA: frame blockIdx.x, channels [32 * blockIdx.y, +32) (lane k owns channel c0 + k in every warp), pixel tile blockIdx.z
// of band_h x band_w.  A sample's taps are separable: its y part (axis_tap of its row coordinate) and its x part.  Per ROI row
// the CTA tabulates the row's ph * gh y parts and pw * gw x parts (the same for every channel), and for every band pixel row y
// and bin row p the window of iy whose y part touches y (likewise x and q); a warp then takes one pixel of the row's bounding
// box at a time, and its 32 lanes walk (p, q, iy, ix) inside the windows, in the contract's order, re-checking each sample.
constexpr int kRoiBwdThreads = 256;
constexpr int kRoiBwdLanes = 32;
constexpr int kRoiBwdLd = kRoiBwdLanes + 1;    // padded rows: conflict-free by channel (gather) and by pixel (NCHW store)
constexpr int kRoiBwdAxis = 256;               // tabulated samples per axis (ph * gh); longer axes are recomputed
constexpr int kRoiBwdSmem = 100 * 1024;        // dynamic shared memory of one CTA: two CTAs per SM
constexpr int kRoiBwdStageBytes = 16 * 1024;   // a row's grad_out chunk is staged when it fits (7x7 bins: 6.3 KB)

__host__ __device__ inline int even_up(long long n) { return (int)((n + 1) & ~1LL); }

__host__ __device__ inline size_t roi_align_bwd_smem(int bh, int bw, int ph, int pw, int staged) {
  return (size_t)(even_up((long long)bh * bw * kRoiBwdLd) + (staged ? even_up((long long)ph * pw * kRoiBwdLd) : 0)) * sizeof(float) +
         (size_t)((long long)bh * ph + (long long)bw * pw + bh + bw) * sizeof(int2);
}

__device__ __forceinline__ AxisTap axis_at(const AxisTap* tab, bool cached, int n, float start, float bin, int grid, int p,
                                           int s) {
  return cached ? tab[p * grid + s] : axis_tap(n, sample_coord(start, p, bin, s, grid));
}

template <typename T>
__device__ __forceinline__ void roi_align_bwd_cta(const T* __restrict__ grad_out, const RoiBwdArgs& a) {
  extern __shared__ __align__(16) float roi_bwd_smem[];
  __shared__ AxisTap ty[kRoiBwdAxis], tx[kRoiBwdAxis];
  __shared__ int rows[kRoiBwdThreads], warp_rows[kRoiBwdThreads / 32], box[4];
  const int H = a.H, W = a.W, ph = a.ph, pw = a.pw, nbins = ph * pw;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int f = blockIdx.x, c0 = blockIdx.y * kRoiBwdLanes;
  const int nbx = (W + a.band_w - 1) / a.band_w;
  const int y0 = (blockIdx.z / nbx) * a.band_h, x0 = (blockIdx.z % nbx) * a.band_w;
  const int bh = min(a.band_h, H - y0), bw = min(a.band_w, W - x0);
  float* acc = roi_bwd_smem;                                                  // [bh * bw][kRoiBwdLd]
  float* gs = acc + even_up((long long)a.band_h * a.band_w * kRoiBwdLd);      // [nbins][kRoiBwdLd] if staged
  int2* ry = reinterpret_cast<int2*>(gs + (a.staged ? even_up((long long)nbins * kRoiBwdLd) : 0));   // [bh][ph]
  int2* rx = ry + a.band_h * ph;                                              // [bw][pw]
  int2* pr = rx + a.band_w * pw;                                              // [bh]: bin rows p with a window on row y
  int2* qr = pr + a.band_h;                                                   // [bw]: bin columns q likewise
  for (int i = tid; i < bh * bw * kRoiBwdLd; i += blockDim.x) acc[i] = 0.0f;
  const int seen = for_each_frame_row(a.rois, a.R, f, rows, warp_rows, [&](int row) {
    const RoiGeom g = roi_geometry(a.rois + 5 * (size_t)row, a.scale, ph, pw, a.sr);
    const int ny = ph * g.gh, nx = pw * g.gw, spb = g.gh * g.gw;
    const bool cy = ny <= kRoiBwdAxis, cx = nx <= kRoiBwdAxis;
    const T* go = grad_out + row * a.go_row;
    if (cy)
      for (int i = tid; i < ny; i += blockDim.x) ty[i] = axis_tap(H, sample_coord(g.start_h, i / g.gh, g.bin_h, i % g.gh, g.gh));
    if (cx)
      for (int i = tid; i < nx; i += blockDim.x) tx[i] = axis_tap(W, sample_coord(g.start_w, i / g.gw, g.bin_w, i % g.gw, g.gw));
    if (a.staged)
      for (int i = tid; i < nbins * kRoiBwdLanes; i += blockDim.x) {
        const int k = a.cl ? i % kRoiBwdLanes : i / nbins, bin = a.cl ? i / kRoiBwdLanes : i % nbins;
        gs[bin * kRoiBwdLd + k] = c0 + k < a.C ? to_f32<T>(go[(long long)bin * a.go_bin + (long long)(c0 + k) * a.go_c]) : 0.0f;
      }
    if (tid == 0) { box[0] = box[2] = 0x7fffffff; box[1] = box[3] = -1; }
    for (int i = tid; i < bh + bw; i += blockDim.x) (i < bh ? pr[i] : qr[i - bh]) = make_int2(0x7fffffff, -1);
    __syncthreads();
    // windows: for band row y and bin row p, [first, last + 1) of the iy whose y part touches y (likewise x, q, ix)
    for (int i = tid; i < bh * ph + bw * pw; i += blockDim.x) {
      const bool isy = i < bh * ph;
      const int j = isy ? i : i - bh * ph, np = isy ? ph : pw;
      const int pix = (isy ? y0 : x0) + j / np, p = j % np, grid = isy ? g.gh : g.gw;
      int lo = grid, hi = 0;
      for (int s = 0; s < grid; ++s) {
        const AxisTap t = isy ? axis_at(ty, cy, H, g.start_h, g.bin_h, g.gh, p, s) : axis_at(tx, cx, W, g.start_w, g.bin_w, g.gw, p, s);
        if (t.lo >= 0 && (t.lo == pix || t.hi == pix)) { lo = min(lo, s); hi = s + 1; }
      }
      (isy ? ry : rx)[j] = make_int2(lo, hi);
      if (hi > lo) {
        atomicMin(&box[isy ? 0 : 2], pix); atomicMax(&box[isy ? 1 : 3], pix);
        int2* pq = isy ? pr + j / np : qr + j / np;
        atomicMin(&pq->x, p); atomicMax(&pq->y, p);
      }
    }
    __syncthreads();
    const int ya = box[0], xa = box[2], nbw = box[3] - box[2] + 1;
    const int items = box[1] < 0 || box[3] < 0 ? 0 : (box[1] - ya + 1) * nbw;
    for (int it = warp; it < items; it += nwarps) {
      const int y = ya + it / nbw, x = xa + it % nbw, yy = y - y0, xx = x - x0;
      float part = 0.0f;
      bool hit = false;
      int slice = 0;
      float* s = acc + (yy * bw + xx) * kRoiBwdLd + lane;
      const int2 prow = pr[yy], qcol = qr[xx];
      for (int p = prow.x; p <= prow.y; ++p) {
        const int2 wy = ry[yy * ph + p];
        if (wy.x >= wy.y) continue;
        for (int q = qcol.x; q <= qcol.y; ++q) {
          const int2 wx = rx[xx * pw + q];
          if (wx.x >= wx.y) continue;
          const int bin = p * pw + q;
          const float gv = a.staged ? gs[bin * kRoiBwdLd + lane]
                                    : (c0 + lane < a.C ? to_f32<T>(go[(long long)bin * a.go_bin + (long long)(c0 + lane) * a.go_c]) : 0.0f);
          for (int iy = wy.x; iy < wy.y; ++iy) {
            const AxisTap ay = axis_at(ty, cy, H, g.start_h, g.bin_h, g.gh, p, iy);
            const bool ylo = ay.lo == y, yhi = ay.hi == y;
            if (ay.lo < 0 || !(ylo || yhi)) continue;
            for (int ix = wx.x; ix < wx.y; ++ix) {
              const AxisTap ax = axis_at(tx, cx, W, g.start_w, g.bin_w, g.gw, q, ix);
              const bool xlo = ax.lo == x, xhi = ax.hi == x;
              if (ax.lo < 0 || !(xlo || xhi)) continue;
              const int sl = (bin * spb + iy * g.gw + ix) / kMaxTaps;
              if (sl != slice) {
                if (hit) *s = __fadd_rn(*s, part);
                part = 0.0f;
                hit = false;
                slice = sl;
              }
              // taps p1 (lo, lo), p2 (lo, hi), p3 (hi, lo), p4 (hi, hi) with make_tap's weights
              if (ylo && xlo) part = __fadd_rn(part, __fdiv_rn(__fmul_rn(gv, __fmul_rn(ay.wlo, ax.wlo)), g.count));
              if (ylo && xhi) part = __fadd_rn(part, __fdiv_rn(__fmul_rn(gv, __fmul_rn(ay.wlo, ax.whi)), g.count));
              if (yhi && xlo) part = __fadd_rn(part, __fdiv_rn(__fmul_rn(gv, __fmul_rn(ay.whi, ax.wlo)), g.count));
              if (yhi && xhi) part = __fadd_rn(part, __fdiv_rn(__fmul_rn(gv, __fmul_rn(ay.whi, ax.whi)), g.count));
              hit = true;
            }
          }
        }
      }
      if (hit) *s = __fadd_rn(*s, part);
    }
    __syncthreads();                            // the tables are rebuilt for the next row
  });
  if (a.mode == kAddIfRows && seen == 0) return;
  __syncthreads();
  roi_bwd_store(a, acc, kRoiBwdLd, f, c0, kRoiBwdLanes, y0, x0, bh, bw);
}

// One kernel body; the three names keep each entry's launches apart in profiles.
__global__ void __launch_bounds__(kRoiBwdThreads) roi_align_bwd_nchw_kernel(const float* __restrict__ grad_out, RoiBwdArgs a) {
  roi_align_bwd_cta<float>(grad_out, a);
}
template <typename T>
__global__ void __launch_bounds__(kRoiBwdThreads) roi_align_bwd_nhwc_kernel(const T* __restrict__ grad_out, RoiBwdArgs a) {
  roi_align_bwd_cta<T>(grad_out, a);
}
template <typename T>
__global__ void __launch_bounds__(kRoiBwdThreads) roi_align_bwd_slice_nhwc_kernel(const T* __restrict__ grad_out, RoiBwdArgs a) {
  roi_align_bwd_cta<T>(grad_out, a);
}

// ---- ROIPool ------------------------------------------------------------------------------------------------------------
// CTA: frame blockIdx.x, a chunk of blockDim.x channels (thread t owns channel c0 + t and, at 32 channels or more,
// shared-memory bank t % 32 of the channels-last accumulator), pixels [band_h * blockIdx.z, +band_h) of the frame.  Every
// thread adds grad_out[row, bin, c] into acc[argmax[row, bin, c] - p0, c] row by row, bin by bin: each element sums its
// contributions in ascending (row, ph, pw) order -- the loop order of torchvision's CPU roi_pool backward.
constexpr int kPoolBwdMaxChunk = 64;           // the smallest chunk and the shared-memory budget: common.cuh
constexpr int kPoolBwdBins = 16;               // bins whose (argmax, gradient) loads are in flight together

template <typename T>
__device__ __forceinline__ void roi_pool_bwd_cta(const T* __restrict__ grad_out, const RoiBwdArgs& a) {
  extern __shared__ __align__(16) float roi_bwd_smem[];
  __shared__ int rows[kPoolBwdMaxChunk], warp_rows[kPoolBwdMaxChunk / 32];
  const int chunk = blockDim.x, tid = threadIdx.x, lda = a.cl ? chunk : chunk + 1;
  const int f = blockIdx.x, c0 = blockIdx.y * chunk, c = c0 + tid, nbins = a.ph * a.pw, npix = a.H * a.W;
  const int p0 = blockIdx.z * a.band_h, npx = min(a.band_h, npix - p0);
  float* acc = roi_bwd_smem;                    // [npx][lda]
  for (int i = tid; i < npx * lda; i += chunk) acc[i] = 0.0f;
  const int seen = for_each_frame_row(a.rois, a.R, f, rows, warp_rows, [&](int row) {
    if (c >= a.C) return;
    const T* g = grad_out + row * a.go_row + (long long)c * a.go_c;
    const int32_t* am = a.argmax + row * a.am_row + (long long)c * a.am_c;
    for (int b0 = 0; b0 < nbins; b0 += kPoolBwdBins) {
      int av[kPoolBwdBins];
      float gv[kPoolBwdBins];
#pragma unroll
      for (int k = 0; k < kPoolBwdBins; ++k) {
        const bool in = b0 + k < nbins;
        av[k] = in ? am[(long long)(b0 + k) * a.am_bin] : -1;
        gv[k] = in ? to_f32<T>(g[(long long)(b0 + k) * a.go_bin]) : 0.0f;
      }
#pragma unroll
      for (int k = 0; k < kPoolBwdBins; ++k)
        if ((unsigned)(av[k] - p0) < (unsigned)npx) {   // -1: empty bin, no contribution
          float* s = acc + (av[k] - p0) * lda + tid;
          *s = __fadd_rn(*s, gv[k]);
        }
    }
  });
  if (a.mode == kAddIfRows && seen == 0) return;
  __syncthreads();
  if (a.cl && a.mode == kAddIfRows) {
    // 16-byte accesses (C and in_ld are multiples of 4 on this path)
    float* dst = a.grad_in + (long long)a.fm.map(f) * a.gi_frame + c0;
    const int nv = min(chunk, a.C - c0) / 4;
    for (int i = tid; i < npx * nv; i += chunk) {
      const int p = i / nv, v = i - p * nv;
      const float4 s = *reinterpret_cast<const float4*>(acc + p * chunk + v * 4);
      float4* d = reinterpret_cast<float4*>(dst + (long long)(p0 + p) * a.gi_pix + v * 4);
      float4 cur = *d;
      cur.x = __fadd_rn(cur.x, s.x); cur.y = __fadd_rn(cur.y, s.y); cur.z = __fadd_rn(cur.z, s.z); cur.w = __fadd_rn(cur.w, s.w);
      *d = cur;
    }
    return;
  }
  roi_bwd_store(a, acc, lda, f, c0, chunk, p0 / a.W, p0 % a.W, 1, npx);
}

__global__ void __launch_bounds__(kPoolBwdMaxChunk) roi_pool_bwd_nchw_kernel(const float* __restrict__ grad_out, RoiBwdArgs a) {
  roi_pool_bwd_cta<float>(grad_out, a);
}
template <typename T>
__global__ void __launch_bounds__(kPoolBwdMaxChunk) roi_pool_bwd_slice_nhwc_kernel(const T* __restrict__ grad_out, RoiBwdArgs a) {
  roi_pool_bwd_cta<T>(grad_out, a);
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)kNumSMs * 32;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

// Chooses the pixel tile (the whole plane when it fits kRoiBwdSmem, else halved rows, then halved columns) and launches
// `kernel` over frames x channel chunks x tiles.
template <typename T>
static int launch_roi_align_bwd(void (*kernel)(const T*, RoiBwdArgs), std::atomic<unsigned long long>& seen, const T* grad_out,
                                RoiBwdArgs a, int frames, cudaStream_t stream, const char* name) {
  if (frames == 0) return 0;
  a.staged = (long long)a.ph * a.pw * kRoiBwdLd * (long long)sizeof(float) <= kRoiBwdStageBytes;
  int bh = a.H, bw = a.W;
  while (roi_align_bwd_smem(bh, bw, a.ph, a.pw, a.staged) > (size_t)kRoiBwdSmem) {
    if (bh > 1) bh = (bh + 1) / 2;
    else if (bw > 1) bw = (bw + 1) / 2;
    else return fail(STEP_E_ARG, "%s: ph=%d x pw=%d bins exceed the shared-memory tables", name, a.ph, a.pw);
  }
  a.band_h = bh;
  a.band_w = bw;
  const dim3 grid(frames, ceil_div(a.C, kRoiBwdLanes), ceil_div(a.H, bh) * ceil_div(a.W, bw));
  if (int rc = allow_dynamic_smem(kernel, seen, kRoiBwdSmem, name)) return rc;
  kernel<<<grid, kRoiBwdThreads, roi_align_bwd_smem(bh, bw, a.ph, a.pw, a.staged), stream>>>(grad_out, a);
  STEP_LAUNCH_CHECK(name);
  return 0;
}

// The widest channel chunk (64 down to 8) whose [H*W, chunk] accumulator fits kPoolBwdSmem, no wider than C needs; planes
// that do not fit even at 8 channels are split into pixel bands.
template <typename T>
static int launch_roi_pool_bwd(void (*kernel)(const T*, RoiBwdArgs), std::atomic<unsigned long long>& seen, const T* grad_out,
                               RoiBwdArgs a, int frames, cudaStream_t stream, const char* name) {
  if (frames == 0) return 0;
  const long long npix = (long long)a.H * a.W;
  int chunk = kPoolBwdMaxChunk;
  while (chunk > kPoolBwdMinChunk && (npix * chunk * (long long)sizeof(float) > kPoolBwdSmem || chunk >= 2 * a.C)) chunk /= 2;
  const int lda = a.cl ? chunk : chunk + 1;
  a.band_h = (int)(npix < kPoolBwdSmem / (lda * (long long)sizeof(float)) ? npix : kPoolBwdSmem / (lda * (long long)sizeof(float)));
  a.band_w = 1;
  const dim3 grid(frames, ceil_div(a.C, chunk), ceil_div(npix, a.band_h));
  if (int rc = allow_dynamic_smem(kernel, seen, kPoolBwdSmem, name)) return rc;
  kernel<<<grid, chunk, (size_t)a.band_h * lda * sizeof(float), stream>>>(grad_out, a);
  STEP_LAUNCH_CHECK(name);
  return 0;
}

}  // namespace step

using namespace step;

extern "C" int step_roi_align_fwd_nchw_f32(const float* feat, int K, int C, int H, int W, const float* rois,
                                           int R, float scale, int ph, int pw, int sampling_ratio, float* out,
                                           step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && C > 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_fwd_nchw: bad shape");
  long long total = (long long)R * C * ph * pw;
  if (total == 0) return 0;  // ROIAlign_cpu.cpp:262-264
  STEP_CHECK_ARG(feat && rois && out, "roi_align_fwd_nchw: null pointer");
  roi_align_fwd_nchw_kernel<<<grid_for(total, 256), 256, 0, cu(stream)>>>(total, feat, scale, C, H, W, ph, pw,
                                                                          sampling_ratio, rois, out);
  STEP_LAUNCH_CHECK("roi_align_fwd_nchw_kernel");
  return 0;
}

extern "C" int step_roi_align_bwd_nchw_f32(const float* grad_out, const float* rois, int R, float scale, int ph,
                                           int pw, int K, int C, int H, int W, int sampling_ratio, float* grad_in,
                                           step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && C > 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_bwd_nchw: bad shape");
  STEP_CHECK_ARG(grad_in, "roi_align_bwd_nchw: null grad_in");
  STEP_CHECK_ARG(R == 0 || (grad_out && rois), "roi_align_bwd_nchw: null pointer");
  static std::atomic<unsigned long long> seen{0};
  // kStore writes every element of the K frames: a frame without a row gets the +0.0f of the reference's zero fill
  return launch_roi_align_bwd(roi_align_bwd_nchw_kernel, seen, grad_out,
                              roi_bwd_args(false, rois, R, scale, ph, pw, sampling_ratio, H, W, C, 0, 0, nullptr, grad_in,
                                           FrameMap{0, 0, 0}, kStore),
                              K, cu(stream), "roi_align_bwd_nchw_kernel");
}

extern "C" int step_roi_pool_fwd_nchw_f32(const float* feat, int K, int C, int H, int W, const float* rois, int R,
                                          float scale, int ph, int pw, float* out, int32_t* argmax,
                                          step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && C > 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_pool_fwd_nchw: bad shape");
  long long total = (long long)R * C * ph * pw;
  if (total == 0) return 0;
  STEP_CHECK_ARG(feat && rois && out && argmax, "roi_pool_fwd_nchw: null pointer");
  roi_pool_fwd_nchw_kernel<<<grid_for(total, 256), 256, 0, cu(stream)>>>(total, feat, scale, C, H, W, ph, pw, rois,
                                                                         out, argmax);
  STEP_LAUNCH_CHECK("roi_pool_fwd_nchw_kernel");
  return 0;
}

extern "C" int step_roi_pool_bwd_nchw_f32(const float* grad_out, const int32_t* argmax, const float* rois, int R,
                                          int ph, int pw, int K, int C, int H, int W, float* grad_in,
                                          step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && C > 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_pool_bwd_nchw: bad shape");
  STEP_CHECK_ARG(grad_in, "roi_pool_bwd_nchw: null grad_in");
  STEP_CHECK_ARG(R == 0 || (grad_out && argmax && rois), "roi_pool_bwd_nchw: null pointer");
  static std::atomic<unsigned long long> seen{0};
  return launch_roi_pool_bwd(roi_pool_bwd_nchw_kernel, seen, grad_out,
                             roi_bwd_args(false, rois, R, 0.0f, ph, pw, 0, H, W, C, 0, 0, argmax, grad_in,
                                          FrameMap{0, 0, 0}, kStore),
                             K, cu(stream), "roi_pool_bwd_nchw_kernel");
}

static int check_nhwc(const char* name, int dtype, int C, int feat_ld, int out_ld, const void* a, const void* b) {
  int vn = dtype == STEP_F16 ? 8 : 4;
  STEP_CHECK_ARG(dtype == STEP_F16 || dtype == STEP_F32, "%s: bad dtype %d", name, dtype);
  STEP_CHECK_ARG(C > 0 && C % vn == 0 && feat_ld % vn == 0 && out_ld % vn == 0 && feat_ld >= C && out_ld >= C,
                 "%s: C=%d feat_ld=%d out_ld=%d must be multiples of %d", name, C, feat_ld, out_ld, vn);
  STEP_CHECK_ARG((((uintptr_t)a | (uintptr_t)b) & 15) == 0, "%s: pointers must be 16-byte aligned", name);
  return 0;
}

extern "C" int step_roi_align_fwd_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                                       const float* rois, int R, float scale, int ph, int pw, int sampling_ratio,
                                       void* out, int out_ld, int roi_T, int feat_T, int t_start, int exact,
                                       step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_fwd_nhwc: bad shape");
  if (R == 0) return 0;
  STEP_CHECK_ARG(feat && rois && out, "roi_align_fwd_nhwc: null pointer");
  if (int rc = check_nhwc("roi_align_fwd_nhwc", dtype, C, feat_ld, out_ld, feat, out)) return rc;
  STEP_CHECK_ARG(roi_T == 0 || (roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T), "roi_align_fwd_nhwc: bad frame map");
  FrameMap fm{roi_T, feat_T, t_start};
  if (dtype == STEP_F16 && exact == 0 && (size_t)ph * pw * sizeof(MergedBin) <= 48 * 1024 &&
      (long long)H * W * feat_ld < (1LL << 31)) {   // table entries hold 32-bit element offsets inside one frame
    // one CTA per ROI row: the row's tap table is built once, in shared memory
    roi_align_fwd_nhwc_f16_packed_kernel<<<R, 256, (size_t)ph * pw * sizeof(MergedBin), cu(stream)>>>(
        (const __half*)feat, H, W, C, feat_ld, rois, scale, ph, pw, sampling_ratio, (__half*)out, out_ld, fm);
    STEP_LAUNCH_CHECK("roi_align_fwd_nhwc_f16_packed_kernel");
    return 0;
  }
  if (dtype == STEP_F16 && exact != 1)
    roi_align_fwd_nhwc_kernel<__half, false><<<R, 256, 0, cu(stream)>>>((const __half*)feat, H, W, C, feat_ld, rois, scale,
                                                                         ph, pw, sampling_ratio, (__half*)out, out_ld, fm);
  else if (dtype == STEP_F16)
    roi_align_fwd_nhwc_kernel<__half, true><<<R, 256, 0, cu(stream)>>>((const __half*)feat, H, W, C, feat_ld, rois, scale,
                                                                        ph, pw, sampling_ratio, (__half*)out, out_ld, fm);
  else
    roi_align_fwd_nhwc_kernel<float, true><<<R, 256, 0, cu(stream)>>>((const float*)feat, H, W, C, feat_ld, rois, scale,
                                                                       ph, pw, sampling_ratio, (float*)out, out_ld, fm);
  STEP_LAUNCH_CHECK("roi_align_fwd_nhwc_kernel");
  return 0;
}

extern "C" int step_roi_pool_fwd_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                                      const float* rois, int R, float scale, int ph, int pw, void* out, int out_ld,
                                      int roi_T, int feat_T, int t_start, step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_pool_fwd_nhwc: bad shape");
  if (R == 0) return 0;
  STEP_CHECK_ARG(feat && rois && out, "roi_pool_fwd_nhwc: null pointer");
  if (int rc = check_nhwc("roi_pool_fwd_nhwc", dtype, C, feat_ld, out_ld, feat, out)) return rc;
  STEP_CHECK_ARG(roi_T == 0 || (roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T), "roi_pool_fwd_nhwc: bad frame map");
  FrameMap fm{roi_T, feat_T, t_start};
  if (dtype == STEP_F16)
    roi_pool_fwd_nhwc_kernel<__half, false><<<R, 256, 0, cu(stream)>>>((const __half*)feat, H, W, C, feat_ld, rois, scale,
                                                                        ph, pw, (__half*)out, out_ld, fm, nullptr);
  else
    roi_pool_fwd_nhwc_kernel<float, false><<<R, 256, 0, cu(stream)>>>((const float*)feat, H, W, C, feat_ld, rois, scale,
                                                                       ph, pw, (float*)out, out_ld, fm, nullptr);
  STEP_LAUNCH_CHECK("roi_pool_fwd_nhwc_kernel");
  return 0;
}

extern "C" int step_roi_pool_fwd_argmax_nhwc(const void* feat, int dtype, int K, int H, int W, int C, int feat_ld,
                                             const float* rois, int R, float scale, int ph, int pw, void* out, int out_ld,
                                             int roi_T, int feat_T, int t_start, int32_t* argmax, step_stream_t stream) {
  STEP_CHECK_ARG(K >= 0 && H > 0 && W > 0 && R >= 0 && ph > 0 && pw > 0, "roi_pool_fwd_argmax_nhwc: bad shape");
  if (R == 0) return 0;
  STEP_CHECK_ARG(feat && rois && out && argmax, "roi_pool_fwd_argmax_nhwc: null pointer");
  if (int rc = check_nhwc("roi_pool_fwd_argmax_nhwc", dtype, C, feat_ld, out_ld, feat, out)) return rc;
  STEP_CHECK_ARG(((uintptr_t)argmax & 15) == 0, "roi_pool_fwd_argmax_nhwc: argmax must be 16-byte aligned");
  STEP_CHECK_ARG((long long)H * W <= kPoolBwdMaxPixels,
                 "roi_pool_fwd_argmax_nhwc: H*W=%lld exceeds the %d-pixel limit of the ROIPool backward's shared-memory accumulator "
                 "(inputs up to ~1280x1280)", (long long)H * W, kPoolBwdMaxPixels);
  STEP_CHECK_ARG(roi_T == 0 || (roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T),
                 "roi_pool_fwd_argmax_nhwc: bad frame map roi_T=%d feat_T=%d t_start=%d", roi_T, feat_T, t_start);
  FrameMap fm{roi_T, feat_T, t_start};
  if (dtype == STEP_F16)
    roi_pool_fwd_nhwc_kernel<__half, true><<<R, 256, 0, cu(stream)>>>((const __half*)feat, H, W, C, feat_ld, rois, scale,
                                                                       ph, pw, (__half*)out, out_ld, fm, argmax);
  else
    roi_pool_fwd_nhwc_kernel<float, true><<<R, 256, 0, cu(stream)>>>((const float*)feat, H, W, C, feat_ld, rois, scale,
                                                                      ph, pw, (float*)out, out_ld, fm, argmax);
  STEP_LAUNCH_CHECK("roi_pool_fwd_argmax_nhwc_kernel");
  return 0;
}

// Channels-last backward entries of the training step (header: step_b200.h).
static int check_bwd_nhwc(const char* name, int dtype, int C, int in_ld, int out_ld) {
  STEP_CHECK_ARG(dtype == STEP_F32 || dtype == STEP_F16, "%s: bad dtype", name);
  STEP_CHECK_ARG(C % 4 == 0 && in_ld % 4 == 0 && out_ld % 4 == 0 && in_ld >= C && out_ld >= C, "%s: C / ld must be multiples of 4", name);
  return 0;
}

extern "C" int step_roi_align_bwd_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                                       int pw, int K, int H, int W, int C, int sampling_ratio, float* grad_in, int in_ld,
                                       step_stream_t stream) {
  STEP_CHECK_ARG(K > 0 && H > 0 && W > 0 && C > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_bwd_nhwc: bad shape");
  if (int rc = check_bwd_nhwc("roi_align_bwd_nhwc", dtype, C, in_ld, out_ld)) return rc;
  STEP_CHECK_ARG(grad_in && (R == 0 || (grad_out && rois)), "roi_align_bwd_nhwc: null pointer");
  STEP_CHECK_ARG((((uintptr_t)grad_in | (uintptr_t)grad_out) & 15) == 0, "roi_align_bwd_nhwc: pointers must be 16-byte aligned");
  const RoiBwdArgs a = roi_bwd_args(true, rois, R, scale, ph, pw, sampling_ratio, H, W, C, out_ld, in_ld, nullptr, grad_in,
                                    FrameMap{0, 0, 0}, kStore);
  static std::atomic<unsigned long long> seen32{0}, seen16{0};
  if (dtype == STEP_F32)
    return launch_roi_align_bwd(roi_align_bwd_nhwc_kernel<float>, seen32, (const float*)grad_out, a, K, cu(stream), "roi_align_bwd_nhwc_kernel");
  return launch_roi_align_bwd(roi_align_bwd_nhwc_kernel<__half>, seen16, (const __half*)grad_out, a, K, cu(stream), "roi_align_bwd_nhwc_kernel");
}

extern "C" size_t step_roi_align_bwd_slice_workspace_bytes(int, int, int, int, int, int) {
  return 0;   // each frame's contribution is formed in shared memory
}

extern "C" int step_roi_align_bwd_slice_nhwc(const void* grad_out, int dtype, int out_ld, const float* rois, int R, float scale, int ph,
                                             int pw, int K, int H, int W, int C, int sampling_ratio, int roi_T, int feat_T, int t_start,
                                             float* grad_in, int in_ld, void* workspace, size_t ws_bytes, step_stream_t stream) {
  (void)workspace; (void)ws_bytes;
  STEP_CHECK_ARG(K > 0 && H > 0 && W > 0 && C > 0 && R >= 0 && ph > 0 && pw > 0, "roi_align_bwd_slice_nhwc: bad shape");
  if (int rc = check_bwd_nhwc("roi_align_bwd_slice_nhwc", dtype, C, in_ld, out_ld)) return rc;
  STEP_CHECK_ARG(feat_T > 0 && K % feat_T == 0 && roi_T > 0 && t_start >= 0 && t_start + roi_T <= feat_T,
                 "roi_align_bwd_slice_nhwc: bad frame map roi_T=%d feat_T=%d t_start=%d K=%d", roi_T, feat_T, t_start, K);
  STEP_CHECK_ARG(grad_in && (R == 0 || (grad_out && rois)), "roi_align_bwd_slice_nhwc: null pointer");
  STEP_CHECK_ARG((((uintptr_t)grad_in | (uintptr_t)grad_out) & 15) == 0, "roi_align_bwd_slice_nhwc: pointers must be 16-byte aligned");
  const RoiBwdArgs a = roi_bwd_args(true, rois, R, scale, ph, pw, sampling_ratio, H, W, C, out_ld, in_ld, nullptr, grad_in,
                                    FrameMap{roi_T, feat_T, t_start}, kAdd);
  const int frames = (K / feat_T) * roi_T;
  static std::atomic<unsigned long long> seen32{0}, seen16{0};
  if (dtype == STEP_F32)
    return launch_roi_align_bwd(roi_align_bwd_slice_nhwc_kernel<float>, seen32, (const float*)grad_out, a, frames, cu(stream),
                                "roi_align_bwd_slice_nhwc_kernel");
  return launch_roi_align_bwd(roi_align_bwd_slice_nhwc_kernel<__half>, seen16, (const __half*)grad_out, a, frames, cu(stream),
                              "roi_align_bwd_slice_nhwc_kernel");
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
  const RoiBwdArgs a = roi_bwd_args(true, rois, R, 0.0f, ph, pw, 0, H, W, C, out_ld, in_ld, argmax, grad_in,
                                    FrameMap{roi_T, feat_T, t_start}, kAddIfRows);
  const int frames = (K / feat_T) * roi_T;
  static std::atomic<unsigned long long> seen32{0}, seen16{0};
  if (dtype == STEP_F32)
    return launch_roi_pool_bwd(roi_pool_bwd_slice_nhwc_kernel<float>, seen32, (const float*)grad_out, a, frames, cu(stream),
                               "roi_pool_bwd_slice_nhwc_kernel");
  return launch_roi_pool_bwd(roi_pool_bwd_slice_nhwc_kernel<__half>, seen16, (const __half*)grad_out, a, frames, cu(stream),
                             "roi_pool_bwd_slice_nhwc_kernel");
}
