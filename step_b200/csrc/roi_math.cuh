// roi_math.cuh -- the ROIAlign sampling of cpu/ROIAlign_cpu.cpp shared by the forward and the backward kernels (roi.cu):
// both must sample the same points for the backward to be the adjoint of the forward.  Every fp32
// operation is explicitly rounded in the reference's operand order; the including files are built with -fmad=false.
#pragma once
#include "common.cuh"

namespace step {

struct Tap {
  int p1, p2, p3, p4;  // pixel offsets (y*W + x); p1 < 0 => sample contributes nothing
  float w1, w2, w3, w4;
};

// One axis of the bilinear tap: the pixels lo, hi (of n along the axis) a sample at coordinate v reads and their weights
// wlo = 1 - l, whi = l.  lo < 0: v is outside [-1, n] and the sample contributes nothing (ROIAlign_cpu.cpp:72-131).
struct AxisTap {
  int lo, hi;
  float wlo, whi;
};

__device__ __forceinline__ AxisTap axis_tap(int n, float v) {
  AxisTap a;
  if (v < -1.0f || v > (float)n) {
    a.lo = a.hi = -1;
    a.wlo = a.whi = 0.0f;
    return a;
  }
  if (v <= 0.0f) v = 0.0f;
  a.lo = (int)v;
  if (a.lo >= n - 1) { a.hi = a.lo = n - 1; v = (float)a.lo; } else { a.hi = a.lo + 1; }
  a.whi = __fsub_rn(v, (float)a.lo);
  a.wlo = __fsub_rn(1.0f, a.whi);
  return a;
}

__device__ __forceinline__ Tap make_tap(int H, int W, float y, float x) {
  Tap t;
  const AxisTap ay = axis_tap(H, y), ax = axis_tap(W, x);
  if (ay.lo < 0 || ax.lo < 0) {
    t.p1 = t.p2 = t.p3 = t.p4 = -1;
    t.w1 = t.w2 = t.w3 = t.w4 = 0.0f;
    return t;
  }
  t.w1 = __fmul_rn(ay.wlo, ax.wlo); t.w2 = __fmul_rn(ay.wlo, ax.whi); t.w3 = __fmul_rn(ay.whi, ax.wlo); t.w4 = __fmul_rn(ay.whi, ax.whi);
  t.p1 = ay.lo * W + ax.lo; t.p2 = ay.lo * W + ax.hi;
  t.p3 = ay.hi * W + ax.lo; t.p4 = ay.hi * W + ax.hi;
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

// Entries of the per-ROI shared-memory tap table of the forward: 7x7 bins x sampling grids up to 4x4; larger grids are
// recomputed.  The backward forms a row's partial sums per kMaxTaps samples (roi.cu).
constexpr int kMaxTaps = 49 * 16;

}  // namespace step
