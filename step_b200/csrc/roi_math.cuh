// roi_math.cuh -- the ROIAlign sampling of cpu/ROIAlign_cpu.cpp shared by the forward kernels (roi.cu) and the backward
// kernels (train.cu): both must sample the same points for the backward to be the adjoint of the forward.  Every fp32
// operation is explicitly rounded in the reference's operand order; the including files are built with -fmad=false.
#pragma once
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

// Entries of the per-ROI shared-memory tap tables: 7x7 bins x sampling grids up to 4x4.  Larger grids are recomputed
// (forward) or processed in slices of this size (backward).
constexpr int kMaxTaps = 49 * 16;

}  // namespace step
