// tubes.cu -- box/tube arithmetic between refinement steps, on device.
//
// Replaces utils/tube_utils.py (decode_coef 165-189, encode_coef 143-163, valid_tubes 59-92,
// extrapolate_tubes 10-27, flatten_tubes 214-246, extend_tubes 248-266) and the per-clip host loop
// of utils/utils.py:87-129 (D->H copy, numpy, per-box Python loop, H->D copy every step).
// All arithmetic is fp32 with explicitly rounded operations in the reference's operand order
// (torch evaluates each line as separate fp32 kernels, so no contraction there either).
// exp/log use CUDA's expf/logf (<= 2 ulp), the only source of non-bit-exactness vs torch CPU.
#include "common.cuh"
#include "tube_math.cuh"

namespace step {

__global__ void tube_decode_kernel(const float* __restrict__ anchors, int astride, const float* __restrict__ deltas,
                                   int n, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) st4(out + 4 * (size_t)i, decode_one(ld4(anchors + (size_t)i * astride), ld4(deltas + 4 * (size_t)i)));
}

__global__ void tube_encode_kernel(const float* __restrict__ gt, const float* __restrict__ anchors, int astride, int n,
                                   float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  st4(out + 4 * (size_t)i, encode_one(ld4(gt + 4 * (size_t)i), ld4(anchors + (size_t)i * astride)));
}

__global__ void tube_valid_kernel(float* __restrict__ boxes, int n, float width, float height) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) st4(boxes + 4 * (size_t)i, valid_one(ld4(boxes + 4 * (size_t)i), width, height));
}

__global__ void tube_extrapolate_kernel(const float* __restrict__ tubes, int n, int L, int T, float width, float height,
                                        float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (tube, component)
  if (i >= n * 4) return;
  int tube = i >> 2, comp = i & 3;
  extrapolate_one(tubes + (size_t)tube * L * 4, L, T, width, height, out + (size_t)tube * (L + 2 * T) * 4, comp);
}

__global__ void tube_extend_kernel(const float* __restrict__ tubes, int n, float ratio, float width, float height,
                                   float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* r = tubes + 5 * (size_t)i;
  CS c = center_size(r[1], r[2], r[3], r[4]);
  float w = __fmul_rn(c.w, ratio), h = __fmul_rn(c.h, ratio);  // tube_utils.py:259-260
  float* o = out + 5 * (size_t)i;
  o[0] = r[0];
  o[1] = fmaxf(__fsub_rn(c.x, __fmul_rn(0.5f, w)), 0.0f);
  o[2] = fmaxf(__fsub_rn(c.y, __fmul_rn(0.5f, h)), 0.0f);
  o[3] = fminf(__fsub_rn(__fadd_rn(c.x, __fmul_rn(0.5f, w)), 1.0f), __fsub_rn(width, 1.0f));
  o[4] = fminf(__fsub_rn(__fadd_rn(c.y, __fmul_rn(0.5f, h)), 1.0f), __fsub_rn(height, 1.0f));
}

// One CTA per tube (blockDim = 64 >= frames handled): decode -> extend -> validate -> re-flatten.
constexpr int kMaxFrames = 64;
__global__ void __launch_bounds__(64) tube_update_kernel(const float* __restrict__ flat_in, const float* __restrict__ loc,
                                                         const float* __restrict__ first, const float* __restrict__ last,
                                                         const int32_t* __restrict__ clip_of_tube, int L, int T,
                                                         int decode_neighbors, int ext_mode, float width, float height,
                                                         float* __restrict__ pred_loc, float* __restrict__ pred_first,
                                                         float* __restrict__ pred_last, float* __restrict__ flat_out) {
  __shared__ float cur[kMaxFrames * 4];   // decoded centre tube [L,4]
  __shared__ float ext[kMaxFrames * 4];   // extended tube [L_out,4]
  const int r = blockIdx.x, t = threadIdx.x;
  const float* fin = flat_in + (size_t)r * L * 5;
  const int L_out = (ext_mode != STEP_EXT_NONE) ? L + 2 * T : L;
  // utils.py:66-70: pred_loc = decode(flat[:,1:], local_loc)
  if (t < L) {
    float4 p = decode_one(ld4(fin + t * 5 + 1), ld4(loc + ((size_t)r * L + t) * 4));
    st4(pred_loc + ((size_t)r * L + t) * 4, p);
    st4(cur + t * 4, p);
  }
  // utils.py:72-79: first/last chunks (frames [0,T) and [L-T,L) of the current tube)
  if (decode_neighbors && t < T) {
    float4 pf = decode_one(ld4(fin + t * 5 + 1), ld4(first + ((size_t)r * T + t) * 4));
    float4 pl = decode_one(ld4(fin + (L - T + t) * 5 + 1), ld4(last + ((size_t)r * T + t) * 4));
    st4(pred_first + ((size_t)r * T + t) * 4, pf);
    st4(pred_last + ((size_t)r * T + t) * 4, pl);
    if (ext_mode == STEP_EXT_PREDICT) {  // utils.py:102-107: cat([first, centre, last], time)
      st4(ext + t * 4, pf);
      st4(ext + (T + L + t) * 4, pl);
    }
  }
  __syncthreads();
  if (ext_mode == STEP_EXT_NONE || ext_mode == STEP_EXT_PREDICT) {
    if (t < L) {
      int dst = (ext_mode == STEP_EXT_PREDICT) ? T + t : t;
      st4(ext + dst * 4, ld4(cur + t * 4));
    }
  } else if (ext_mode == STEP_EXT_EXTRAPOLATE) {
    // utils.py:109-112: extrapolate_tubes(cur, T) with its default 400x400 clamp (tube_utils.py:10)
    if (t < 4) extrapolate_one(cur, L, T, 400.0f, 400.0f, ext, t);
  } else {  // STEP_EXT_MEAN, utils.py:114-118: np.mean over time (fp32 pairwise in numpy; L is tiny)
    if (t < 4) {
      float s = 0.0f;
      for (int k = 0; k < L; ++k) s = __fadd_rn(s, cur[k * 4 + t]);
      float m = __fdiv_rn(s, (float)L);
      for (int k = 0; k < T; ++k) { ext[k * 4 + t] = m; ext[(T + L + k) * 4 + t] = m; }
      for (int k = 0; k < L; ++k) ext[(T + k) * 4 + t] = cur[k * 4 + t];
    }
  }
  __syncthreads();
  // utils.py:121 valid_tubes(image_size) then 127-129 flatten_tubes(batch_idx=True)
  if (t < L_out) {
    float4 v = valid_one(ld4(ext + t * 4), width, height);
    float* o = flat_out + ((size_t)r * L_out + t) * 5;
    o[0] = (float)(clip_of_tube[r] * L_out + t);  // tube_utils.py:238 arange(T) + i*T
    o[1] = v.x; o[2] = v.y; o[3] = v.z; o[4] = v.w;
  }
}

}  // namespace step

using namespace step;

extern "C" int step_tube_decode_f32(const float* anchors, int anchor_stride, const float* deltas, int n, float* out,
                                    step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0 && anchor_stride >= 4, "tube_decode: bad n/stride");
  if (n == 0) return 0;
  STEP_CHECK_ARG(anchors && deltas && out, "tube_decode: null pointer");
  tube_decode_kernel<<<ceil_div(n, 128), 128, 0, cu(stream)>>>(anchors, anchor_stride, deltas, n, out);
  STEP_LAUNCH_CHECK("tube_decode_kernel");
  return 0;
}

extern "C" int step_tube_encode_f32(const float* gt, const float* anchors, int anchor_stride, int n, float* out,
                                    step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0 && anchor_stride >= 4, "tube_encode: bad n/stride");
  if (n == 0) return 0;
  STEP_CHECK_ARG(gt && anchors && out, "tube_encode: null pointer");
  tube_encode_kernel<<<ceil_div(n, 128), 128, 0, cu(stream)>>>(gt, anchors, anchor_stride, n, out);
  STEP_LAUNCH_CHECK("tube_encode_kernel");
  return 0;
}

extern "C" int step_tube_valid_f32(float* boxes, int n, float width, float height, step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0, "tube_valid: bad n");
  if (n == 0) return 0;
  STEP_CHECK_ARG(boxes, "tube_valid: null pointer");
  tube_valid_kernel<<<ceil_div(n, 128), 128, 0, cu(stream)>>>(boxes, n, width, height);
  STEP_LAUNCH_CHECK("tube_valid_kernel");
  return 0;
}

extern "C" int step_tube_extrapolate_f32(const float* tubes, int n, int L, int T, float width, float height,
                                         float* out, step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0 && L >= 1 && T >= 2 && L >= T, "tube_extrapolate: need L >= T >= 2");
  if (n == 0) return 0;
  STEP_CHECK_ARG(tubes && out, "tube_extrapolate: null pointer");
  tube_extrapolate_kernel<<<ceil_div(n * 4, 128), 128, 0, cu(stream)>>>(tubes, n, L, T, width, height, out);
  STEP_LAUNCH_CHECK("tube_extrapolate_kernel");
  return 0;
}

extern "C" int step_tube_extend_f32(const float* tubes, int n, float ratio, float width, float height, float* out,
                                    step_stream_t stream) {
  STEP_CHECK_ARG(n >= 0, "tube_extend: bad n");
  if (n == 0) return 0;
  STEP_CHECK_ARG(tubes && out, "tube_extend: null pointer");
  tube_extend_kernel<<<ceil_div(n, 128), 128, 0, cu(stream)>>>(tubes, n, ratio, width, height, out);
  STEP_LAUNCH_CHECK("tube_extend_kernel");
  return 0;
}

extern "C" int step_tube_update_f32(const float* flat_in, const float* loc, const float* first, const float* last,
                                    const int32_t* clip_of_tube, int R, int L, int T, int decode_neighbors,
                                    int ext_mode, float width, float height, float* pred_loc, float* pred_first,
                                    float* pred_last, float* flat_out, step_stream_t stream) {
  STEP_CHECK_ARG(R >= 0 && L >= 1 && T >= 1 && T <= L, "tube_update: bad R/L/T");
  STEP_CHECK_ARG(ext_mode >= STEP_EXT_NONE && ext_mode <= STEP_EXT_MEAN, "tube_update: bad ext_mode");
  STEP_CHECK_ARG(L + (ext_mode ? 2 * T : 0) <= kMaxFrames, "tube_update: more than %d frames", kMaxFrames);
  STEP_CHECK_ARG(ext_mode != STEP_EXT_PREDICT || decode_neighbors, "tube_update: PREDICT needs decode_neighbors");
  STEP_CHECK_ARG(ext_mode != STEP_EXT_EXTRAPOLATE || T >= 2, "tube_update: EXTRAPOLATE needs T >= 2");
  if (R == 0) return 0;
  STEP_CHECK_ARG(flat_in && loc && clip_of_tube && pred_loc && flat_out, "tube_update: null pointer");
  STEP_CHECK_ARG(!decode_neighbors || (first && last && pred_first && pred_last), "tube_update: null neighbor ptr");
  tube_update_kernel<<<R, 64, 0, cu(stream)>>>(flat_in, loc, first, last, clip_of_tube, L, T, decode_neighbors,
                                               ext_mode, width, height, pred_loc, pred_first, pred_last, flat_out);
  STEP_LAUNCH_CHECK("tube_update_kernel");
  return 0;
}
