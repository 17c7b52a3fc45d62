// tube_math.cuh -- per-box tube arithmetic of utils/tube_utils.py shared by tubes.cu (the inference loop), select.cu
// (train_select), train.cu (the regression targets of the losses) and nms.cu (the detection boxes).
#pragma once
#include "common.cuh"

namespace step {

__device__ __forceinline__ float4 valid_one(float4 b, float width, float height) {
  // tube_utils.py:72-88: clamp, then degenerate boxes become the whole image
  b.x = fmaxf(0.0f, b.x); b.y = fmaxf(0.0f, b.y);
  b.z = fminf(width, b.z); b.w = fminf(height, b.w);
  if (!(b.x < __fsub_rn(b.z, 2.0f) && b.y < __fsub_rn(b.w, 2.0f))) { b.x = 0.0f; b.y = 0.0f; b.z = width; b.w = height; }
  return b;
}

__device__ __forceinline__ float4 ld4(const float* p) { return make_float4(p[0], p[1], p[2], p[3]); }
__device__ __forceinline__ void st4(float* p, float4 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w; }

struct CS { float x, y, w, h; };

__device__ __forceinline__ CS center_size(float x1, float y1, float x2, float y2) {
  // tube_utils.py:136-139
  CS c;
  c.w = __fadd_rn(__fsub_rn(x2, x1), 1.0f);
  c.h = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
  c.x = __fadd_rn(x1, __fmul_rn(0.5f, c.w));
  c.y = __fadd_rn(y1, __fmul_rn(0.5f, c.h));
  return c;
}

__device__ __forceinline__ float4 decode_one(float4 a, float4 d) {
  // tube_utils.py:176-187
  CS c = center_size(a.x, a.y, a.z, a.w);
  float px = __fadd_rn(__fmul_rn(c.w, d.x), c.x);
  float py = __fadd_rn(__fmul_rn(c.h, d.y), c.y);
  float pw = __fmul_rn(c.w, expf(d.z));
  float ph = __fmul_rn(c.h, expf(d.w));
  float4 o;
  o.x = __fsub_rn(px, __fmul_rn(0.5f, pw));
  o.y = __fsub_rn(py, __fmul_rn(0.5f, ph));
  o.z = __fsub_rn(__fadd_rn(px, __fmul_rn(0.5f, pw)), 1.0f);
  o.w = __fsub_rn(__fadd_rn(py, __fmul_rn(0.5f, ph)), 1.0f);
  return o;
}

__device__ __forceinline__ float4 encode_one(float4 g, float4 a) {
  // tube_utils.py:143-163 encode_coef(gt, anchor) -> (dx, dy, dw, dh)
  CS cg = center_size(g.x, g.y, g.z, g.w), ca = center_size(a.x, a.y, a.z, a.w);
  return make_float4(__fdiv_rn(__fsub_rn(cg.x, ca.x), ca.w), __fdiv_rn(__fsub_rn(cg.y, ca.y), ca.h),
                     logf(__fdiv_rn(cg.w, ca.w)), logf(__fdiv_rn(cg.h, ca.h)));
}

// linear recurrence of tube_utils.py:18-20; coefficients are Python doubles multiplied into fp32
// arrays (numpy casts the python scalar to fp32 first), so a = fl32(T/(T-1)), b = fl32(1/(T-1)).
__device__ __forceinline__ void extrapolate_one(const float* __restrict__ in /*[L,4]*/, int L, int T, float width,
                                                float height, float* __restrict__ out /*[L+2T,4]*/, int comp) {
  const float a = (float)((double)T / (double)(T - 1)), b = (float)(1.0 / (double)(T - 1));
  const int Lo = L + 2 * T;
  for (int t = 0; t < L; ++t) out[(T + t) * 4 + comp] = in[t * 4 + comp];
  for (int i = 0; i < T; ++i) {
    // new[-T+i] = a*new[-T+i-1] - b*new[-T+i-T];  new[T-i-1] = a*new[T-i] - b*new[T-i+T-1]
    int hi = Lo - T + i;
    out[hi * 4 + comp] = __fsub_rn(__fmul_rn(a, out[(hi - 1) * 4 + comp]), __fmul_rn(b, out[(hi - T) * 4 + comp]));
    int lo = T - i - 1;
    out[lo * 4 + comp] = __fsub_rn(__fmul_rn(a, out[(lo + 1) * 4 + comp]), __fmul_rn(b, out[(lo + T) * 4 + comp]));
  }
  for (int t = 0; t < Lo; ++t) {  // tube_utils.py:22-25
    float v = out[t * 4 + comp];
    if (comp == 0 || comp == 1) v = fmaxf(0.0f, v);
    else if (comp == 2) v = fminf(__fsub_rn(width, 1.0f), v);
    else v = fminf(__fsub_rn(height, 1.0f), v);
    out[t * 4 + comp] = v;
  }
}

}  // namespace step
