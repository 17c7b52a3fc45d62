// clip_prep.cu -- the reference's BaseTransform and TubeAugmentation on the device: uint8 frames -> fp32 clip [B,T,3,H,W]
// in one launch (step_frames_to_clip_u8 and step_frames_to_clip_aug_u8, include/step_b200.h).  Compiled with
// -fmad=false: every product and sum below is rounded on its own, in the order cv2's generic float32 code uses, and the
// few operations cv2's compiled code fuses are written as __fmaf_rn, so the result is bit-identical to it.
//
// One CTA writes a tile of kTileW output columns x kTileH output rows of one frame, all 3 channels.  The source rows and
// columns the tile taps are staged in shared memory as uint8 (each source line is read from L2 once per CTA); the
// conversion to float goes through a 256-entry table.  When the tile's source rows do not fit the stage at once (strong
// vertical downscale) the tile's rows are processed in groups.
//
// The augmenting instantiation (kAug) stages the same way, in the crop's mirrored coordinates: the tile taps the crop
// rect of the source, read right to left when the clip is flipped.  Every augmentation step before the resize is per
// pixel, so it is applied to each staged pixel the tile taps (aug_pixel) instead of through the table: the photometric
// program (its HSV round trip mixes the channels), the channel permutation, ConvertFromInts and the erase regions.
#include <cfloat>

#include "common.cuh"

namespace step {
namespace {

constexpr int kTileW = 128;               // output columns per CTA: one 512-byte fp32 row segment per (channel, row)
constexpr int kTileH = 16;                // output rows per CTA
constexpr int kThreads = 256;
constexpr int kStageBytes = 40 * 1024;    // uint8 source rows x 3 channels x tile source columns
constexpr int kMaxWidthRatio = 48;        // W0 <= 48 W keeps one group of 2 rows within the stage: see the header

struct Taps {
  int s0, s1;
  float f;
};

// cv2 resize.cpp (INTER_LINEAR): fx = (float)((dx + 0.5) * scale - 0.5), scale = 1 / ((double)dst / src); sx = floor(fx),
// fx -= sx.  Columns clamp the tap and zero the weight at both ends; rows keep the unclamped weight and only clamp the
// taps (its vertical pass clips the row index), which is what makes the border rows differ from a replicated row.
__device__ __forceinline__ Taps linear_taps(int d, int n_dst, int n_src, bool clamp_weight) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn((double)n_dst, (double)n_src));
  float f = (float)__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  Taps t;
  if (clamp_weight) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= n_src - 1) s = n_src - 1, f = 0.f;
    t.s0 = s;
  } else {
    t.s0 = min(max(s, 0), n_src - 1);
  }
  t.s1 = min(max(s + 1, 0), n_src - 1);
  t.f = f;
  return t;
}

// INTER_AREA's fast path taps rows/columns 2d and 2d + 1
__device__ __forceinline__ Taps taps(int d, int n_dst, int n_src, bool area, bool is_col) {
  if (area) return Taps{2 * d, 2 * d + 1, 0.f};
  return linear_taps(d, n_dst, n_src, is_col);
}

struct Bgr {
  float b, g, r;
};

__device__ __forceinline__ float pick(const Bgr& x, int k) { return k == 0 ? x.b : k == 1 ? x.g : x.r; }

// ConvertFromInts on an fp32 value: scale 2 is u*2/255 - 1 (each step rounded), 1 is u/255, 0 leaves it
__device__ __forceinline__ float convert(float u, int scale_mode) {
  return scale_mode == 2 ? __fsub_rn(__fdiv_rn(__fmul_rn(u, 2.f), 255.f), 1.f) : scale_mode == 1 ? __fdiv_rn(u, 255.f) : u;
}

// PhotometricDistort on one BGR pixel, with cv2 4.x's float HSV arithmetic: BGR2HSV's hue is fma(num, 60 / (diff + eps),
// offset), with 360 folded into the red sector's offset in its 8-lane loop; its scalar loop, which takes the last W0 % 8
// pixels of a source row (`tail`), adds 360 after the fma where the hue is negative.  HSV2BGR fuses 1 - s*f and
// 1 - s*(1 - f).
__device__ __forceinline__ Bgr photometric(Bgr x, const step_clip_aug& p, bool tail) {
  if (p.brightness) x = Bgr{__fadd_rn(x.b, p.brightness_delta), __fadd_rn(x.g, p.brightness_delta),
                            __fadd_rn(x.r, p.brightness_delta)};
  if (p.contrast && p.contrast_first)
    x = Bgr{__fmul_rn(x.b, p.contrast_alpha), __fmul_rn(x.g, p.contrast_alpha), __fmul_rn(x.r, p.contrast_alpha)};
  // BGR2HSV
  const float v = fmaxf(fmaxf(x.r, x.g), x.b);
  const float diff = __fsub_rn(v, fminf(fminf(x.r, x.g), x.b));
  float s = __fdiv_rn(diff, __fadd_rn(fabsf(v), FLT_EPSILON));
  const float d = __fdiv_rn(60.f, __fadd_rn(diff, FLT_EPSILON));
  float num, offset;
  if (x.r == v) {
    num = __fsub_rn(x.g, x.b);
    offset = num < 0.f && !tail ? 360.f : 0.f;
  } else if (x.g == v) {
    num = __fsub_rn(x.b, x.r);
    offset = 120.f;
  } else {
    num = __fsub_rn(x.r, x.g);
    offset = 240.f;
  }
  float h = __fmaf_rn(num, d, offset);
  if (tail && h < 0.f) h = __fadd_rn(h, 360.f);
  if (p.saturation) s = __fmul_rn(s, p.saturation_alpha);
  if (p.hue) {  // the reference's wrap: subtract where above 360, then add where below 0
    h = __fadd_rn(h, p.hue_delta);
    if (h > 360.f) h = __fsub_rn(h, 360.f);
    if (h < 0.f) h = __fadd_rn(h, 360.f);
  }
  // HSV2BGR
  const float h6 = __fmul_rn(h, 6.f / 360.f);
  const float pre = truncf(h6), f = __fsub_rn(h6, pre);
  const int sector = (int)__fsub_rn(pre, __fmul_rn(truncf(__fmul_rn(pre, 1.f / 6.f)), 6.f));
  const float t1 = __fmul_rn(v, __fsub_rn(1.f, s));
  const float t2 = __fmul_rn(v, __fmaf_rn(-s, f, 1.f));
  const float t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, f), 1.f));
  switch (sector) {
    case 0: x = Bgr{t1, t3, v}; break;
    case 1: x = Bgr{t1, v, t2}; break;
    case 2: x = Bgr{t3, v, t1}; break;
    case 3: x = Bgr{v, t2, t1}; break;
    case 4: x = Bgr{v, t1, t3}; break;
    default: x = Bgr{t2, t1, v}; break;
  }
  if (p.contrast && !p.contrast_first)
    x = Bgr{__fmul_rn(x.b, p.contrast_alpha), __fmul_rn(x.g, p.contrast_alpha), __fmul_rn(x.r, p.contrast_alpha)};
  return x;
}

// Every augmentation step before the resize, on the staged source pixel at (xs, ys) of the mirrored crop: `px` points
// at its R value, with the G and B values `wc` and 2 wc bytes further (the stage holds the source's RGB channel order).
// Returns the BGR value the reference's frame holds there after RandomErase.
__device__ __forceinline__ Bgr aug_pixel(const uint8_t* px, int wc, int xs, int ys, bool tail, const step_clip_aug& p,
                                         const float* lut, int scale_mode, const step_aug_erase* __restrict__ erase,
                                         const float* __restrict__ noise) {
  const uint8_t ub = px[2 * wc], ug = px[wc], ur = px[0];
  Bgr x;
  if (p.photometric) {
    x = photometric(Bgr{(float)ub, (float)ug, (float)ur}, p, tail);
    x = Bgr{pick(x, p.perm[0]), pick(x, p.perm[1]), pick(x, p.perm[2])};
    if (scale_mode == 2)  // np.clip on the distorted floats
      x = Bgr{fminf(fmaxf(x.b, 0.f), 255.f), fminf(fmaxf(x.g, 0.f), 255.f), fminf(fmaxf(x.r, 0.f), 255.f)};
    x = Bgr{convert(x.b, scale_mode), convert(x.g, scale_mode), convert(x.r, scale_mode)};
  } else {
    x = Bgr{lut[ub], lut[ug], lut[ur]};
  }
  for (int e = p.erase_count - 1; e >= 0; --e) {  // the later region is on top
    const step_aug_erase r = erase[p.erase_begin + e];
    if (xs >= r.x1 && xs < r.x2 && ys >= r.y1 && ys < r.y2) {
      const float* n = noise + r.noise + ((long long)(ys - r.y1) * (r.x2 - r.x1) + (xs - r.x1)) * 3;
      return Bgr{__ldg(n), __ldg(n + 1), __ldg(n + 2)};
    }
  }
  return x;
}

template <bool kAug>
__global__ void __launch_bounds__(kThreads, 3) frames_to_clip_u8_kernel(const step_frame_src* __restrict__ table,
                                                                     const step_clip_aug* __restrict__ params,
                                                                     const step_aug_erase* __restrict__ erase,
                                                                     const float* __restrict__ noise, int T, int H,
                                                                     int W, int scale_mode, float3 mean, float3 stdv,
                                                                     float* __restrict__ out) {
  __shared__ uint8_t stage[kStageBytes];
  __shared__ float lut[256];
  __shared__ int col0[kTileW], col1[kTileW];
  __shared__ float colw0[kTileW], colw1[kTileW];
  __shared__ int row0[kTileH], row1[kTileH];
  __shared__ float roww0[kTileH], roww1[kTileH];

  const int tid = threadIdx.x;
  const int bt = blockIdx.z, b = bt / T, t = bt % T;
  const step_frame_src src = table[b];
  step_clip_aug p{};
  if constexpr (kAug) p = params[b];
  // the resize's source: the crop rect for the augmenting kernel, the whole frame otherwise
  const int H0 = kAug ? p.h : src.H0, W0 = kAug ? p.w : src.W0;
  const bool area = H0 == 2 * H && W0 == 2 * W;  // cv2 resizes an exact 2x downscale as INTER_AREA
  const int x_begin = blockIdx.x * kTileW, y_begin = blockIdx.y * kTileH;
  const int nx = min(kTileW, W - x_begin), ny = min(kTileH, H - y_begin);
  float* out_f = out + (long long)bt * 3 * H * W;
  // (v - 0) / 1 == v exactly, so I3D's means 0 and stds 1 skip the division
  const bool identity = mean.x == 0.f && mean.y == 0.f && mean.z == 0.f && stdv.x == 1.f && stdv.y == 1.f && stdv.z == 1.f;

  static_assert(kThreads == 256, "one table entry per thread");
  {
    const float u = (float)tid;
    lut[tid] = scale_mode == 2 ? __fsub_rn(__fdiv_rn(__fmul_rn(u, 2.f), 255.f), 1.f)
             : scale_mode == 1 ? __fdiv_rn(u, 255.f) : u;
  }
  if (tid < nx) {
    const Taps c = taps(x_begin + tid, W, W0, area, true);
    col0[tid] = c.s0; col1[tid] = c.s1;
    colw0[tid] = __fsub_rn(1.f, c.f); colw1[tid] = c.f;
  }
  if (tid >= kTileW && tid - kTileW < ny) {
    const int i = tid - kTileW;
    const Taps r = taps(y_begin + i, H, H0, area, false);
    row0[i] = r.s0; row1[i] = r.s1;
    roww0[i] = __fsub_rn(1.f, r.f); roww1[i] = r.f;
  }
  __syncthreads();

  const int ca = col0[0], wc = col1[nx - 1] - ca + 1;
  const int rows_cap = kStageBytes / (3 * wc);
  if (rows_cap < 2) {  // outside the documented W0 <= 48 W: mark the tile instead of reading past the stage
    for (int k = tid; k < 3 * ny * kTileW; k += kThreads) {
      const int i = k % kTileW, rc = k / kTileW;
      if (i < nx) out_f[((long long)(rc % 3) * H + y_begin + rc / 3) * W + x_begin + i] = __int_as_float(0x7fc00000);
    }
    return;
  }

  // stage column x holds source column x0 + ca + x, or x0 + w - 1 - ca - x for a mirrored crop
  const long long col_step = kAug && p.flip ? -src.stride_w : src.stride_w;
  const int col_base = kAug ? (p.flip ? p.x0 + p.w - 1 - ca : p.x0 + ca) : ca;
  const uint8_t* frame = src.data + (long long)t * src.stride_t + (long long)(kAug ? p.y0 : 0) * src.stride_h +
                         (long long)col_base * src.stride_w;
  const int i = tid % kTileW;
  for (int g0 = 0; g0 < ny;) {
    const int ra = row0[g0];
    int g1 = g0 + 1;
    while (g1 < ny && row1[g1] - ra + 1 <= rows_cap) ++g1;
    const int nr = row1[g1 - 1] - ra + 1;

    // stage rows ra .. ra+nr-1, channels 0..2, columns ca .. ca+wc-1: one warp per (row, channel) line.  The staging is
    // load-latency bound, so with unit column stride (a stacked [B,T,3,H0,W0] batch) the aligned middle of a line is read
    // as 4-byte words; the unaligned ends, and other strides, byte by byte.
    const int lane = tid % 32;
    for (int line = tid / 32; line < nr * 3; line += kThreads / 32) {
      const uint8_t* lp = frame + (long long)(ra + line / 3) * src.stride_h + (long long)(line % 3) * src.stride_c;
      uint8_t* s = stage + line * wc;
      if (col_step == 1) {
        const int head = min(wc, (int)((4 - ((uintptr_t)lp & 3)) & 3));
        const int nw = (wc - head) / 4, tail = head + 4 * nw;
        const uint32_t* pw = reinterpret_cast<const uint32_t*>(lp + head);
        if (lane < head) s[lane] = __ldg(lp + lane);
        if (lane < wc - tail) s[tail + lane] = __ldg(lp + tail + lane);
#pragma unroll 4
        for (int k = lane; k < nw; k += 32) {
          const uint32_t v = __ldg(pw + k);
          uint8_t* d = s + head + 4 * k;
          d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24);
        }
      } else {
#pragma unroll 8
        for (int x = lane; x < wc; x += 32) s[x] = __ldg(lp + (long long)x * col_step);
      }
    }
    __syncthreads();

    if (kAug && i < nx) {
      const int xs0 = col0[i], xs1 = col1[i];
      const float wx0 = colw0[i], wx1 = colw1[i];
      // cv2's BGR2HSV runs its scalar loop over the last W0 % 8 pixels of each source row
      const int tail_from = src.W0 - src.W0 % 8;
      const bool tail0 = (p.flip ? p.x0 + p.w - 1 - xs0 : p.x0 + xs0) >= tail_from;
      const bool tail1 = (p.flip ? p.x0 + p.w - 1 - xs1 : p.x0 + xs1) >= tail_from;
      for (int j = g0 + tid / kTileW; j < g1; j += kThreads / kTileW) {
        const int ys0 = row0[j], ys1 = row1[j];
        const uint8_t* s0 = stage + (ys0 - ra) * 3 * wc;
        const uint8_t* s1 = stage + (ys1 - ra) * 3 * wc;
        const Bgr a = aug_pixel(s0 + xs0 - ca, wc, xs0, ys0, tail0, p, lut, scale_mode, erase, noise);
        const Bgr bb = aug_pixel(s0 + xs1 - ca, wc, xs1, ys0, tail1, p, lut, scale_mode, erase, noise);
        const Bgr cc = aug_pixel(s1 + xs0 - ca, wc, xs0, ys1, tail0, p, lut, scale_mode, erase, noise);
        const Bgr d = aug_pixel(s1 + xs1 - ca, wc, xs1, ys1, tail1, p, lut, scale_mode, erase, noise);
#pragma unroll
        for (int c = 0; c < 3; ++c) {  // output channel c is the frame's BGR channel 2 - c (the dataset's swap)
          const int k = 2 - c;
          const float va = pick(a, k), vb = pick(bb, k), vc = pick(cc, k), vd = pick(d, k);
          float v;
          if (area) {
            v = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(va, vb), vc), vd), 0.25f);
          } else {
            const float h0 = __fadd_rn(__fmul_rn(va, wx0), __fmul_rn(vb, wx1));
            const float h1 = __fadd_rn(__fmul_rn(vc, wx0), __fmul_rn(vd, wx1));
            v = __fadd_rn(__fmul_rn(h0, roww0[j]), __fmul_rn(h1, roww1[j]));
          }
          if (!identity) {
            const float m = c == 0 ? mean.x : c == 1 ? mean.y : mean.z, sd = c == 0 ? stdv.x : c == 1 ? stdv.y : stdv.z;
            v = __fdiv_rn(__fsub_rn(v, m), sd);
          }
          out_f[((long long)c * H + y_begin + j) * W + x_begin + i] = v;
        }
      }
    }
    if (!kAug && i < nx) {
      const int x0 = col0[i] - ca, x1 = col1[i] - ca;
      const float wx0 = colw0[i], wx1 = colw1[i];
      for (int k = tid / kTileW; k < 3 * (g1 - g0); k += kThreads / kTileW) {
        const int c = k % 3, j = g0 + k / 3;
        const uint8_t* s0 = stage + ((row0[j] - ra) * 3 + c) * wc;
        const uint8_t* s1 = stage + ((row1[j] - ra) * 3 + c) * wc;
        const float a = lut[s0[x0]], bb = lut[s0[x1]], cc = lut[s1[x0]], d = lut[s1[x1]];
        float v;
        if (area) {
          v = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(a, bb), cc), d), 0.25f);
        } else {
          const float h0 = __fadd_rn(__fmul_rn(a, wx0), __fmul_rn(bb, wx1));
          const float h1 = __fadd_rn(__fmul_rn(cc, wx0), __fmul_rn(d, wx1));
          v = __fadd_rn(__fmul_rn(h0, roww0[j]), __fmul_rn(h1, roww1[j]));
        }
        if (!identity) {
          const float m = c == 0 ? mean.x : c == 1 ? mean.y : mean.z, sd = c == 0 ? stdv.x : c == 1 ? stdv.y : stdv.z;
          v = __fdiv_rn(__fsub_rn(v, m), sd);
        }
        out_f[((long long)c * H + y_begin + j) * W + x_begin + i] = v;
      }
    }
    __syncthreads();
    g0 = g1;
  }
}

}  // namespace
}  // namespace step

extern "C" int step_frames_to_clip_u8(const step_frame_src* table, int B, int T, int H, int W, int scale_mode,
                                      const float* mean3, const float* std3, float* out, step_stream_t stream) {
  using namespace step;
  STEP_CHECK_ARG(table && mean3 && std3 && out, "frames_to_clip_u8: null pointer (table %p, mean3 %p, std3 %p, out %p)",
                 (const void*)table, (const void*)mean3, (const void*)std3, (const void*)out);
  STEP_CHECK_ARG(B > 0 && T > 0 && H > 0 && W > 0, "frames_to_clip_u8: sizes must be positive (B %d, T %d, H %d, W %d)", B,
                 T, H, W);
  STEP_CHECK_ARG(scale_mode >= 0 && scale_mode <= 2, "frames_to_clip_u8: scale_mode %d is not 0, 1 or 2", scale_mode);
  STEP_CHECK_ARG((long long)B * T <= 65535, "frames_to_clip_u8: B*T = %lld frames exceeds 65535", (long long)B * T);
  static_assert(kStageBytes / (3 * ((kTileW - 1) * kMaxWidthRatio + 3)) >= 2, "stage too small for W0 <= 48 W");
  dim3 grid(ceil_div(W, kTileW), ceil_div(H, kTileH), B * T);
  frames_to_clip_u8_kernel<false><<<grid, kThreads, 0, cu(stream)>>>(table, nullptr, nullptr, nullptr, T, H, W, scale_mode,
                                                              make_float3(mean3[0], mean3[1], mean3[2]),
                                                              make_float3(std3[0], std3[1], std3[2]), out);
  STEP_LAUNCH_CHECK("frames_to_clip_u8_kernel");
  return 0;
}

extern "C" int step_frames_to_clip_aug_u8(const step_frame_src* table, const step_clip_aug* params,
                                          const step_aug_erase* erase, const float* noise, int B, int T, int H, int W,
                                          int scale_mode, const float* mean3, const float* std3, float* out,
                                          step_stream_t stream) {
  using namespace step;
  STEP_CHECK_ARG(table && params && mean3 && std3 && out,
                 "frames_to_clip_aug_u8: null pointer (table %p, params %p, mean3 %p, std3 %p, out %p)", (const void*)table,
                 (const void*)params, (const void*)mean3, (const void*)std3, (const void*)out);
  STEP_CHECK_ARG(!erase == !noise, "frames_to_clip_aug_u8: erase %p and noise %p must both be set or both be null",
                 (const void*)erase, (const void*)noise);
  STEP_CHECK_ARG(B > 0 && T > 0 && H > 0 && W > 0, "frames_to_clip_aug_u8: sizes must be positive (B %d, T %d, H %d, W %d)",
                 B, T, H, W);
  STEP_CHECK_ARG(scale_mode >= 0 && scale_mode <= 2, "frames_to_clip_aug_u8: scale_mode %d is not 0, 1 or 2", scale_mode);
  STEP_CHECK_ARG((long long)B * T <= 65535, "frames_to_clip_aug_u8: B*T = %lld frames exceeds 65535", (long long)B * T);
  dim3 grid(ceil_div(W, kTileW), ceil_div(H, kTileH), B * T);
  frames_to_clip_u8_kernel<true><<<grid, kThreads, 0, cu(stream)>>>(table, params, erase, noise, T, H, W, scale_mode,
                                                                     make_float3(mean3[0], mean3[1], mean3[2]),
                                                                     make_float3(std3[0], std3[1], std3[2]), out);
  STEP_LAUNCH_CHECK("frames_to_clip_aug_u8_kernel");
  return 0;
}
