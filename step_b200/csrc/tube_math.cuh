// tube_math.cuh -- per-box tube arithmetic shared by tubes.cu (the inference loop) and select.cu (train_select).
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
