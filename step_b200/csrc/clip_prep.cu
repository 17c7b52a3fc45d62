// clip_prep.cu -- the reference's BaseTransform on the device: uint8 frames -> fp32 clip [B,T,3,H,W] in one launch
// (step_frames_to_clip_u8, include/step_b200.h).  Compiled with -fmad=false: every product and sum below is rounded on
// its own, in the order cv2's generic float32 resize uses, so the result is bit-identical to it.
//
// One CTA writes a tile of kTileW output columns x kTileH output rows of one frame, all 3 channels.  The source rows and
// columns the tile taps are staged in shared memory as uint8 (each source line is read from L2 once per CTA); the
// conversion to float goes through a 256-entry table.  When the tile's source rows do not fit the stage at once (strong
// vertical downscale) the tile's rows are processed in groups.
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

__global__ void __launch_bounds__(kThreads, 3) frames_to_clip_u8_kernel(const step_frame_src* __restrict__ table, int T, int H,
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
  const int H0 = src.H0, W0 = src.W0;
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

  const uint8_t* frame = src.data + (long long)t * src.stride_t + (long long)ca * src.stride_w;
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
      const uint8_t* p = frame + (long long)(ra + line / 3) * src.stride_h + (long long)(line % 3) * src.stride_c;
      uint8_t* s = stage + line * wc;
      if (src.stride_w == 1) {
        const int head = min(wc, (int)((4 - ((uintptr_t)p & 3)) & 3));
        const int nw = (wc - head) / 4, tail = head + 4 * nw;
        const uint32_t* pw = reinterpret_cast<const uint32_t*>(p + head);
        if (lane < head) s[lane] = __ldg(p + lane);
        if (lane < wc - tail) s[tail + lane] = __ldg(p + tail + lane);
#pragma unroll 4
        for (int k = lane; k < nw; k += 32) {
          const uint32_t v = __ldg(pw + k);
          uint8_t* d = s + head + 4 * k;
          d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24);
        }
      } else {
#pragma unroll 8
        for (int x = lane; x < wc; x += 32) s[x] = __ldg(p + (long long)x * src.stride_w);
      }
    }
    __syncthreads();

    if (i < nx) {
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
  frames_to_clip_u8_kernel<<<grid, kThreads, 0, cu(stream)>>>(table, T, H, W, scale_mode,
                                                              make_float3(mean3[0], mean3[1], mean3[2]),
                                                              make_float3(std3[0], std3[1], std3[2]), out);
  STEP_LAUNCH_CHECK("frames_to_clip_u8_kernel");
  return 0;
}
