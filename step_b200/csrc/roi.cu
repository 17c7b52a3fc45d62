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
#include "common.cuh"

namespace step {

struct Tap {
  int p1, p2, p3, p4;  // pixel offsets (y*W + x); p1 < 0 => sample contributes nothing
  float w1, w2, w3, w4;
};

__device__ __forceinline__ Tap make_tap(int H, int W, float y, float x) {
  Tap t;
  // ROIAlign_cpu.cpp:72-131
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) {
    t.p1 = t.p2 = t.p3 = t.p4 = -1;
    t.w1 = t.w2 = t.w3 = t.w4 = 0.0f;
    return t;
  }
  if (y <= 0.0f) y = 0.0f;
  if (x <= 0.0f) x = 0.0f;
  int y_low = (int)y, x_low = (int)x, y_high, x_high;
  if (y_low >= H - 1) { y_high = y_low = H - 1; y = (float)y_low; } else { y_high = y_low + 1; }
  if (x_low >= W - 1) { x_high = x_low = W - 1; x = (float)x_low; } else { x_high = x_low + 1; }
  float ly = __fsub_rn(y, (float)y_low), lx = __fsub_rn(x, (float)x_low);
  float hy = __fsub_rn(1.0f, ly), hx = __fsub_rn(1.0f, lx);
  t.w1 = __fmul_rn(hy, hx); t.w2 = __fmul_rn(hy, lx); t.w3 = __fmul_rn(ly, hx); t.w4 = __fmul_rn(ly, lx);
  t.p1 = y_low * W + x_low;  t.p2 = y_low * W + x_high;
  t.p3 = y_high * W + x_low; t.p4 = y_high * W + x_high;
  return t;
}

struct RoiGeom {
  int batch, gh, gw;
  float start_w, start_h, bin_h, bin_w, count;
};

__device__ __forceinline__ RoiGeom roi_geometry(const float* __restrict__ roi, float scale, int ph, int pw,
                                                int sampling_ratio) {
  RoiGeom g;
  // ROIAlign_cpu.cpp:163-191
  g.batch = (int)roi[0];
  g.start_w = __fmul_rn(roi[1], scale);
  g.start_h = __fmul_rn(roi[2], scale);
  float end_w = __fmul_rn(roi[3], scale), end_h = __fmul_rn(roi[4], scale);
  float rw = fmaxf(__fsub_rn(end_w, g.start_w), 1.0f);
  float rh = fmaxf(__fsub_rn(end_h, g.start_h), 1.0f);
  g.bin_h = __fdiv_rn(rh, (float)ph);
  g.bin_w = __fdiv_rn(rw, (float)pw);
  g.gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(rh, (float)ph));
  g.gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(__fdiv_rn(rw, (float)pw));
  g.count = (float)(g.gh * g.gw);
  return g;
}

__device__ __forceinline__ float sample_coord(float start, int p, float bin, int i, int grid) {
  // ROIAlign_cpu.cpp:62-64: start + p*bin + (i + .5)*bin / grid
  return __fadd_rn(__fadd_rn(start, __fmul_rn((float)p, bin)),
                   __fdiv_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), bin), (float)grid));
}

__device__ __forceinline__ float tap_dot(const Tap& t, float v1, float v2, float v3, float v4) {
  // ROIAlign_cpu.cpp:225-228  w1*v1 + w2*v2 + w3*v3 + w4*v4, left to right, no contraction
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t.w1, v1), __fmul_rn(t.w2, v2)), __fmul_rn(t.w3, v3)),
                   __fmul_rn(t.w4, v4));
}

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

// cuda/ROIAlign_cuda.cu:201-278 (float atomicAdd scatter, like the reference)
__global__ void __launch_bounds__(256) roi_align_bwd_nchw_kernel(long long total, const float* __restrict__ gout,
                                                                 float scale, int C, int H, int W, int ph,
                                                                 int pw, int sampling_ratio,
                                                                 const float* __restrict__ rois,
                                                                 float* __restrict__ gin) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int q = (int)(idx % pw);
    int p = (int)((idx / pw) % ph);
    int c = (int)((idx / pw / ph) % C);
    int n = (int)(idx / pw / ph / C);
    RoiGeom g = roi_geometry(rois + 5 * (size_t)n, scale, ph, pw, sampling_ratio);
    float* plane = gin + ((size_t)g.batch * C + c) * H * W;
    float top = gout[idx];
    for (int iy = 0; iy < g.gh; ++iy) {
      float y = sample_coord(g.start_h, p, g.bin_h, iy, g.gh);
      for (int ix = 0; ix < g.gw; ++ix) {
        float x = sample_coord(g.start_w, q, g.bin_w, ix, g.gw);
        Tap t = make_tap(H, W, y, x);
        if (t.p1 < 0) continue;
        atomicAdd(plane + t.p1, __fdiv_rn(__fmul_rn(top, t.w1), g.count));
        atomicAdd(plane + t.p2, __fdiv_rn(__fmul_rn(top, t.w2), g.count));
        atomicAdd(plane + t.p3, __fdiv_rn(__fmul_rn(top, t.w3), g.count));
        atomicAdd(plane + t.p4, __fdiv_rn(__fmul_rn(top, t.w4), g.count));
      }
    }
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

__global__ void __launch_bounds__(256) roi_pool_bwd_nchw_kernel(long long total, const float* __restrict__ gout,
                                                                const int32_t* __restrict__ argmax, int C,
                                                                int H, int W, int ph, int pw,
                                                                const float* __restrict__ rois,
                                                                float* __restrict__ gin) {
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int c = (int)((idx / pw / ph) % C);
    int n = (int)(idx / pw / ph / C);
    int batch = (int)rois[5 * (size_t)n];
    int a = argmax[idx];
    if (a != -1) atomicAdd(gin + ((size_t)batch * C + c) * H * W + a, gout[idx]);  // ROIPool_cuda.cu:125-129
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

constexpr int kMaxTaps = 49 * 16;  // 7x7 bins, up to 4x4 samples per bin in smem; larger grids recompute

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
                                                 int out_ld, int part, int parts) {
  // this CTA handles channel vectors [cv0, cv0 + cnt) of every V-th of the row (blockIdx.y = part): small batches of
  // ROIs (704 rows in the pipeline) are split over `parts` CTAs per row so that the gather is not one short wave
  const int hv = nvec / V;
  const int cnt = hv / parts, cv0 = part * cnt;
  int bin = threadIdx.x / cnt, cv = threadIdx.x - bin * cnt;   // incremental (bin, cv): no per-item division
  const int dbin = blockDim.x / cnt, dcv = blockDim.x - dbin * cnt;
  const __half2 z2 = __float2half2_rn(0.0f);
  while (bin < nbins) {
    const MergedBin& b = bins[bin];
    __half2 acc[V][4];
#pragma unroll
    for (int u = 0; u < V; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = z2;
    const __half* fp = fbase + (cv0 + cv) * 8;
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
    __half* op = obase + (size_t)bin * out_ld + (cv0 + cv) * 8;
#pragma unroll
    for (int u = 0; u < V; ++u) *reinterpret_cast<uint4*>(op + u * hv * 8) = *reinterpret_cast<const uint4*>(acc[u]);
    bin += dbin; cv += dcv;
    if (cv >= cnt) { cv -= cnt; ++bin; }
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
  __half* obase = out + (size_t)r * nbins * out_ld;
  const int nvec = C >> 3;
  const int part = blockIdx.y, parts = gridDim.y;
  // Distinct pixels one bin can touch, per axis: g + 1 when its g samples are at most one pixel apart (the bin is no wider
  // than g pixels, always so for the adaptive grid), else two per sample.
  const int nh = g.bin_h <= (float)g.gh ? g.gh + 1 : 2 * g.gh, nw = g.bin_w <= (float)g.gw ? g.gw + 1 : 2 * g.gw;
  if (nh * nw > kMaxMerged) {
    // a bin may not fit the table (sampling grid > 3x3, or a fixed sampling_ratio with bins wider than the grid):
    // direct form with fp32 FMAs, no table
    const float ic = 1.0f / g.count;
    const int pv = nvec / parts, pv0 = part * pv;
    for (int item = threadIdx.x; item < nbins * pv; item += blockDim.x) {
      const int bin = item / pv, cv = pv0 + item - bin * pv;
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
  if ((nvec & 1) == 0) roi_gather_items<2>(bins, nbins, nvec, fbase, obase, out_ld, part, parts);
  else roi_gather_items<1>(bins, nbins, nvec, fbase, obase, out_ld, part, parts);
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

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)kNumSMs * 32;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
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
  cudaError_t e = cudaMemsetAsync(grad_in, 0, sizeof(float) * (size_t)K * C * H * W, cu(stream));
  if (e != cudaSuccess) return fail((int)e, "roi_align_bwd_nchw: memset: %s", cudaGetErrorString(e));
  long long total = (long long)R * C * ph * pw;
  if (total == 0) return 0;
  STEP_CHECK_ARG(grad_out && rois, "roi_align_bwd_nchw: null pointer");
  roi_align_bwd_nchw_kernel<<<grid_for(total, 256), 256, 0, cu(stream)>>>(total, grad_out, scale, C, H, W, ph, pw,
                                                                          sampling_ratio, rois, grad_in);
  STEP_LAUNCH_CHECK("roi_align_bwd_nchw_kernel");
  return 0;
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
  cudaError_t e = cudaMemsetAsync(grad_in, 0, sizeof(float) * (size_t)K * C * H * W, cu(stream));
  if (e != cudaSuccess) return fail((int)e, "roi_pool_bwd_nchw: memset: %s", cudaGetErrorString(e));
  long long total = (long long)R * C * ph * pw;
  if (total == 0) return 0;
  STEP_CHECK_ARG(grad_out && argmax && rois, "roi_pool_bwd_nchw: null pointer");
  roi_pool_bwd_nchw_kernel<<<grid_for(total, 256), 256, 0, cu(stream)>>>(total, grad_out, argmax, C, H, W, ph, pw,
                                                                         rois, grad_in);
  STEP_LAUNCH_CHECK("roi_pool_bwd_nchw_kernel");
  return 0;
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
    // One CTA per ROI row by default.  Splitting a row's channels over several CTAs (STEP_B200_ROI_PARTS=2|4, kept for A/B)
    // makes every part rebuild the row's tap table.
    int parts = 1;
    if (const char* e = getenv("STEP_B200_ROI_PARTS")) {
      const int nvec = C / 8, hv = (nvec & 1) == 0 ? nvec / 2 : nvec, v = atoi(e);
      if (v >= 1 && hv % v == 0 && nvec % v == 0) parts = v;
    }
    roi_align_fwd_nhwc_f16_packed_kernel<<<dim3(R, parts), 128 * (parts > 1 ? 1 : 2), (size_t)ph * pw * sizeof(MergedBin), cu(stream)>>>(
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
