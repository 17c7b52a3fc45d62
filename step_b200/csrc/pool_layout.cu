// pool_layout.cu -- HBM-bound channels-last kernels: TF-SAME max pooling, layout conversion at the
// module boundary, small reductions and the small-N linear layers of the head.
//
// MaxPool3dTFPadding (models/i3dpt.py:114-126) = ConstantPad3d(0) + MaxPool3d(ceil_mode=True):
// the padded cells hold 0 (not -inf), and windows may hang over the *padded* extent (ceil mode),
// where they see nothing.  Everything is 16-byte vectorised along C.
#include <stdlib.h>

#include "common.cuh"

namespace step {

// Thread mapping is the whole optimisation: a CTA owns a compact (TT x TH x TW) tile of output pixels and
// a 64-byte channel chunk (CV = 4 vectors), thread = (pixel, vector).  The 27 taps of neighbouring
// outputs then hit the same few KB in L1 instead of re-reading L2 27 times (the pools of
// Mixed.branch_3, i3dpt.py:150-153, are 3x3x3 / stride 1).  Padded cells hold 0 (ConstantPad3d), cells
// beyond the padded extent (ceil_mode overhang) are ignored.
template <typename T> __device__ __forceinline__ uint4 vec_lowest();
template <> __device__ __forceinline__ uint4 vec_lowest<float>() {
  const uint32_t v = __float_as_uint(-3.402823466e+38f);
  return make_uint4(v, v, v, v);
}
template <> __device__ __forceinline__ uint4 vec_lowest<__half>() {
  return make_uint4(0xFBFFFBFFu, 0xFBFFFBFFu, 0xFBFFFBFFu, 0xFBFFFBFFu);  // -65504 in both halves
}
template <typename T> __device__ __forceinline__ uint4 vec_max(uint4 a, uint4 b);
template <> __device__ __forceinline__ uint4 vec_max<float>(uint4 a, uint4 b) {
  return make_uint4(__float_as_uint(fmaxf(__uint_as_float(a.x), __uint_as_float(b.x))),
                    __float_as_uint(fmaxf(__uint_as_float(a.y), __uint_as_float(b.y))),
                    __float_as_uint(fmaxf(__uint_as_float(a.z), __uint_as_float(b.z))),
                    __float_as_uint(fmaxf(__uint_as_float(a.w), __uint_as_float(b.w))));
}
__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
  __half2 r = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
  return *reinterpret_cast<uint32_t*>(&r);
}
template <> __device__ __forceinline__ uint4 vec_max<__half>(uint4 a, uint4 b) {
  return make_uint4(hmax2_u32(a.x, b.x), hmax2_u32(a.y, b.y), hmax2_u32(a.z, b.z), hmax2_u32(a.w, b.w));
}
// kPoolCV vectors of 16 B per pixel per CTA: 8 (= one full 128-byte line: a 64-byte chunk made two CTAs pull the
// same DRAM line, 2x read traffic in the ncu capture) when the channel count allows, else 4.
template <typename T, int CKT, int CKH, int CKW, int kPoolCV>
__global__ void __launch_bounds__(256) maxpool3d_kernel(const T* __restrict__ x, int N, int T_, int H, int W, int C,
                                                        int in_ld, int KT_, int KH_, int KW_, int ST, int SH, int SW,
                                                        int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                                                        int pad_hi_w, int OT, int OH, int OW, T* __restrict__ y,
                                                        int out_ld, int TT, int TH, int TW) {
  constexpr int VN = Vec16<T>::N;
  // compile-time window (fully unrolled: all tap loads are issued back to back) or runtime window (CK* == 0)
  const int KT = CKT ? CKT : KT_, KH = CKH ? CKH : KH_, KW = CKW ? CKW : KW_;
  const int nvec = C / VN;
  const int tiles_w = (OW + TW - 1) / TW, tiles_h = (OH + TH - 1) / TH, tiles_t = (OT + TT - 1) / TT;
  int r = blockIdx.x;
  const int w0 = (r % tiles_w) * TW; r /= tiles_w;
  const int h0 = (r % tiles_h) * TH; r /= tiles_h;
  const int t0 = (r % tiles_t) * TT;
  const int n = r / tiles_t;
  const int cv = blockIdx.y * kPoolCV + (threadIdx.x % kPoolCV);
  if (cv >= nvec) return;
  const int npix = TT * TH * TW;
  for (int p = threadIdx.x / kPoolCV; p < npix; p += blockDim.x / kPoolCV) {
    const int ow = w0 + p % TW, oh = h0 + (p / TW) % TH, ot = t0 + p / (TW * TH);
    if (ow >= OW || oh >= OH || ot >= OT) continue;
    // max is exact in the storage type: stay in packed half2 (4 HMNMX2 per 16-byte load, no converts)
    uint4 m = vec_lowest<T>();
    bool touches_pad = false, any = false;
#pragma unroll
    for (int kt = 0; kt < KT; ++kt) {
      const int t = ot * ST + kt - PT;          // coordinate in the un-padded tensor
      if (t >= T_ + pad_hi_t) continue;         // beyond the padded extent (ceil_mode overhang)
      const bool tp = (t < 0) || (t >= T_);
#pragma unroll
      for (int kh = 0; kh < KH; ++kh) {
        const int h = oh * SH + kh - PH;
        if (h >= H + pad_hi_h) continue;
        if (tp || h < 0 || h >= H) { touches_pad = true; continue; }
        const T* rowp = x + (((size_t)n * T_ + t) * H + h) * W * in_ld + cv * VN;
#pragma unroll
        for (int kw = 0; kw < KW; ++kw) {
          const int w = ow * SW + kw - PW;
          if (w >= W + pad_hi_w) continue;
          if (w < 0 || w >= W) { touches_pad = true; continue; }
          m = vec_max<T>(m, *reinterpret_cast<const uint4*>(rowp + (size_t)w * in_ld));
          any = true;
        }
      }
    }
    if (touches_pad || !any) m = vec_max<T>(m, make_uint4(0, 0, 0, 0));  // +0.0 in both fp32 and fp16
    *reinterpret_cast<uint4*>(y + ((((size_t)n * OT + ot) * OH + oh) * OW + ow) * out_ld + cv * VN) = m;
  }
}

// 3x3x3 / stride 1 / pad 1 (Mixed.branch_3, i3dpt.py:150-153) on maps whose width is a multiple of 7 (112/16 .. 7),
// separable and marching along t: a thread owns a 7-pixel row segment x one 16-byte channel vector and walks TS output
// planes.  For every input plane it loads the 3 x 9 neighbourhood once, reduces it over (h, w) into a
// 7-vector P[tt], and emits out[t] = max(P[t-1], P[t], P[t+1]) from two carried 7-vectors: 27 loads and 70 vector
// maxima per plane instead of 81 and 182 per output row.  The kernel is latency bound on the small maps, so the host
// picks TS to keep ~50k threads in flight.
template <typename T>
__global__ void __launch_bounds__(128) maxpool3d_333_march_kernel(const T* __restrict__ x, int N, int T_, int H, int W, int C,
                                                                  int in_ld, T* __restrict__ y, int out_ld, int TS) {
  constexpr int VN = Vec16<T>::N, WB = 7;
  const int nvec = C / VN, wsegs = W / WB, tsegs = (T_ + TS - 1) / TS;
  const long long total = (long long)N * tsegs * H * wsegs * nvec;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % nvec);
  long long r = idx / nvec;
  const int ws = (int)(r % wsegs); r /= wsegs;
  const int h = (int)(r % H); r /= H;
  const int ts = (int)(r % tsegs);
  const int n = (int)(r / tsegs);
  const int w0 = ws * WB, t0 = ts * TS, t1 = min(T_, t0 + TS);
  const bool wl = w0 > 0, wr = w0 + WB < W;
  const uint4 lo = vec_lowest<T>();
  uint4 p1[WB], m2[WB];
#pragma unroll
  for (int j = 0; j < WB; ++j) { p1[j] = lo; m2[j] = lo; }
  for (int tt = t0 - 1; tt <= t1; ++tt) {
    uint4 pc[WB];
#pragma unroll
    for (int j = 0; j < WB; ++j) pc[j] = lo;
    if (tt >= 0 && tt < T_) {
      uint4 v[3][WB + 2];
#pragma unroll
      for (int dh = 0; dh < 3; ++dh) {
        const int hh = h + dh - 1;
        const bool hv = hh >= 0 && hh < H;
        const T* rowp = x + ((((size_t)n * T_ + tt) * H + (hv ? hh : h)) * W + w0) * in_ld + cv * VN;
        v[dh][0] = (hv && wl) ? *reinterpret_cast<const uint4*>(rowp - in_ld) : lo;
#pragma unroll
        for (int j = 0; j < WB; ++j) v[dh][j + 1] = hv ? *reinterpret_cast<const uint4*>(rowp + (size_t)j * in_ld) : lo;
        v[dh][WB + 1] = (hv && wr) ? *reinterpret_cast<const uint4*>(rowp + (size_t)WB * in_ld) : lo;
      }
#pragma unroll
      for (int j = 0; j < WB + 2; ++j) v[0][j] = vec_max<T>(v[0][j], vec_max<T>(v[1][j], v[2][j]));
#pragma unroll
      for (int j = 0; j < WB; ++j) pc[j] = vec_max<T>(v[0][j], vec_max<T>(v[0][j + 1], v[0][j + 2]));
    }
    const int t = tt - 1;
    if (t >= t0) {
      // windows that overlap the zero padding see a 0 (ConstantPad3d, i3dpt.py:120)
      const bool edge_th = (t == 0) || (t == T_ - 1) || (h == 0) || (h == H - 1);
      T* orow = y + ((((size_t)n * T_ + t) * H + h) * W + w0) * out_ld + cv * VN;
#pragma unroll
      for (int j = 0; j < WB; ++j) {
        uint4 m = vec_max<T>(m2[j], pc[j]);
        if (edge_th || (w0 + j == 0) || (w0 + j == W - 1)) m = vec_max<T>(m, make_uint4(0, 0, 0, 0));
        *reinterpret_cast<uint4*>(orow + (size_t)j * out_ld) = m;
      }
    }
#pragma unroll
    for (int j = 0; j < WB; ++j) { m2[j] = vec_max<T>(p1[j], pc[j]); p1[j] = pc[j]; }
  }
}


// Strided windows ((1,3,3)/(1,2,2) after the stem and conv 2c, (3,3,3)/(2,2,2) between mixed_3 and mixed_4,
// i3dpt.py:191-209) with the same separable marching scheme: a thread owns WB consecutive outputs of one row and one
// 16-byte channel vector, reduces every input plane it needs over (h, w) ONCE into a WB-vector, carries the KT - ST
// planes two consecutive outputs share, and emits max over the KT planes.  Zero padding / ceil-mode overhang follow
// maxpool3d_kernel above: a window that overlaps the zero padding in any dimension sees a 0.
__device__ __forceinline__ bool pool_pad_tap(int o, int S, int P, int K, int D, int pad_hi) {
  bool z = false;
  for (int k = 0; k < K; ++k) {
    const int pos = o * S + k - P;
    z = z || pos < 0 || (pos >= D && pos < D + pad_hi);
  }
  return z;
}

template <typename T, int KT, int KH, int KW, int ST, int SH, int SW, int WB>
__global__ void __launch_bounds__(128) maxpool3d_march_kernel(const T* __restrict__ x, int N, int T_, int H, int W, int C,
                                                              int in_ld, int PT, int PH, int PW, int pad_hi_t, int pad_hi_h,
                                                              int pad_hi_w, int OT, int OH, int OW, T* __restrict__ y,
                                                              int out_ld, int TS) {
  constexpr int VN = Vec16<T>::N, NC = (WB - 1) * SW + KW, CARRY = KT > ST ? KT - ST : 0;
  const int nvec = C / VN, wsegs = (OW + WB - 1) / WB, tsegs = (OT + TS - 1) / TS;
  const long long total = (long long)N * tsegs * OH * wsegs * nvec;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % nvec);
  long long r = idx / nvec;
  const int ws = (int)(r % wsegs); r /= wsegs;
  const int oh = (int)(r % OH); r /= OH;
  const int ts = (int)(r % tsegs);
  const int n = (int)(r / tsegs);
  const int ow0 = ws * WB, ot0 = ts * TS, ot1 = min(OT, ot0 + TS);
  const int wbase = ow0 * SW - PW, hbase = oh * SH - PH;
  const uint4 lo = vec_lowest<T>();
  const bool zh = pool_pad_tap(oh, SH, PH, KH, H, pad_hi_h);
  bool zw[WB];
#pragma unroll
  for (int j = 0; j < WB; ++j) zw[j] = pool_pad_tap(ow0 + j, SW, PW, KW, W, pad_hi_w);

  // one input plane reduced over the (KH x KW) window of each of the WB outputs
  auto plane = [&](int tt, uint4* dst) {
#pragma unroll
    for (int j = 0; j < WB; ++j) dst[j] = lo;
    if (tt < 0 || tt >= T_) return;
#pragma unroll
    for (int dh = 0; dh < KH; ++dh) {
      const int hh = hbase + dh;
      if (hh < 0 || hh >= H) continue;
      const T* rowp = x + (((size_t)n * T_ + tt) * H + hh) * W * in_ld + cv * VN;
      uint4 v[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int w = wbase + c;
        v[c] = (w >= 0 && w < W) ? *reinterpret_cast<const uint4*>(rowp + (size_t)w * in_ld) : lo;
      }
#pragma unroll
      for (int j = 0; j < WB; ++j) {
        uint4 m = v[j * SW];
#pragma unroll
        for (int dw = 1; dw < KW; ++dw) m = vec_max<T>(m, v[j * SW + dw]);
        dst[j] = vec_max<T>(dst[j], m);
      }
    }
  };

  uint4 pl[KT][WB];
#pragma unroll
  for (int i = 0; i < CARRY; ++i) plane(ot0 * ST - PT + i, pl[i]);
  for (int ot = ot0; ot < ot1; ++ot) {
    const int tbase = ot * ST - PT;
#pragma unroll
    for (int i = CARRY; i < KT; ++i) plane(tbase + i, pl[i]);
    const bool z = zh || pool_pad_tap(ot, ST, PT, KT, T_, pad_hi_t);
    T* orow = y + ((((size_t)n * OT + ot) * OH + oh) * OW + ow0) * out_ld + cv * VN;
#pragma unroll
    for (int j = 0; j < WB; ++j) {
      uint4 m = pl[0][j];
#pragma unroll
      for (int i = 1; i < KT; ++i) m = vec_max<T>(m, pl[i][j]);
      if (z || zw[j]) m = vec_max<T>(m, make_uint4(0, 0, 0, 0));
      if (ow0 + j < OW) *reinterpret_cast<uint4*>(orow + (size_t)j * out_ld) = m;
    }
#pragma unroll
    for (int i = 0; i < CARRY; ++i)
#pragma unroll
      for (int j = 0; j < WB; ++j) pl[i][j] = pl[i + ST][j];
  }
}

// x [A,B,P,C] (C contiguous, pixel stride ld, row a at a * a_stride) -> y [A, P*C]  (mean over B, fp32 accumulate in
// index order)
template <typename TI, typename TO>
__global__ void mean_mid_kernel(const TI* __restrict__ x, int A, int B, int P, int C, int ld, long long a_stride,
                                TO* __restrict__ y) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)A * P * C) return;
  int c = (int)(idx % C);
  int p = (int)((idx / C) % P);
  int a = (int)(idx / ((long long)C * P));
  float s = 0.0f;
  for (int b = 0; b < B; ++b) s += to_f32<TI>(x[(size_t)a * a_stride + ((size_t)b * P + p) * ld + c]);
  y[idx] = from_f32<TO>(s / (float)B);
}

// fp16 input, 8 channels per thread (16-byte loads); the per-channel sums run in the same index order as above
template <typename TO>
__global__ void mean_mid_h8_kernel(const __half* __restrict__ x, int A, int B, int P, int C, int ld, long long a_stride,
                                   TO* __restrict__ y) {
  const int cv = C >> 3;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)A * P * cv) return;
  const int c = (int)(idx % cv) * 8;
  const int p = (int)((idx / cv) % P);
  const int a = (int)(idx / ((long long)cv * P));
  float s[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = 0.0f;
  for (int b = 0; b < B; ++b) {
    float v[8];
    load16(x + (size_t)a * a_stride + ((size_t)b * P + p) * ld + c, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] += v[k];
  }
  TO* o = y + ((size_t)a * P + p) * C + c;
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = from_f32<TO>(s[k] / (float)B);
}

// clip [N,T,Cc,H,W] fp32 -> [N,T,H,W,ld]
template <typename T>
__global__ void clip_to_ndhwc_kernel(const float* __restrict__ clip, int N, int T_, int Cc, int H, int W,
                                     T* __restrict__ out, int ld) {
  long long total = (long long)N * T_ * H * W;
  for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
       pix += (long long)gridDim.x * blockDim.x) {
    long long hw = pix % ((long long)H * W);
    long long nt = pix / ((long long)H * W);
    T* o = out + (size_t)pix * ld;
    for (int c = 0; c < ld; ++c)
      o[c] = from_f32<T>(c < Cc ? clip[((size_t)nt * Cc + c) * H * W + hw] : 0.0f);
  }
}

// clip [N,T,Cc,H,W] fp32 -> s2d [N,T/2,H/2,W/2,ld] f16, channel ((rt*2+rh)*2+rw)*Cc + c.
// One CTA per output row (n, t2, h2): the 4*Cc input rows it needs are read coalesced into smem, then
// each thread emits one 16-byte (8-channel) vector of one output pixel: both sides fully coalesced.
constexpr int kS2dRows = 1;   // output rows per CTA (8 was slower: fewer CTAs hide less latency)
__global__ void __launch_bounds__(256) clip_to_s2d_kernel(const float* __restrict__ clip, int N, int T_, int Cc, int H,
                                                          int W, __half* __restrict__ out, int ld) {
  extern __shared__ float rows[];  // [rt][rh][c][W]
  __shared__ int ch_off[64];       // output channel -> offset into rows[] (row base + rw), -1 for padding channels
  const int T2 = T_ / 2, H2 = H / 2, W2 = W / 2;
  int r = blockIdx.x;
  const int h2 = r % H2; r /= H2;
  const int t2 = r % T2;
  const int n = r / T2;
  const int nvec = ld / 8;
  // channel ch = ((rt*2+rh)*2+rw)*Cc + c  ->  smem row (rt,rh,c), column 2*w2+rw.  One runtime div/mod per
  // CHANNEL (first ld threads) instead of eight per thread: the kernel was issue-bound on that setup.
  if (threadIdx.x < ld && threadIdx.x < 64) {
    const int ch = threadIdx.x;
    int off = -1;
    if (ch < 8 * Cc) { const int c = ch % Cc, q = ch / Cc; off = ((q >> 1) * Cc + c) * W + (q & 1); }
    ch_off[ch] = off;
  }
  for (int rt = 0; rt < 2; ++rt)
    for (int rh = 0; rh < 2; ++rh)
      for (int c = 0; c < Cc; ++c) {
        const float* src = clip + ((((size_t)n * T_ + 2 * t2 + rt) * Cc + c) * H + 2 * h2 + rh) * W;
        float* dst = rows + ((rt * 2 + rh) * Cc + c) * W;
        for (int w = threadIdx.x; w < W; w += blockDim.x) dst[w] = src[w];
      }
  __syncthreads();
  const int cvs = threadIdx.x % nvec;          // blockDim.x is a multiple of nvec (ld = 32 -> 4)
  int offs[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) offs[k] = ch_off[cvs * 8 + k];
  __half* orow = out + (((size_t)n * T2 + t2) * H2 + h2) * W2 * ld;
  for (int w2 = threadIdx.x / nvec; w2 < W2; w2 += blockDim.x / nvec) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = offs[k] >= 0 ? rows[offs[k] + 2 * w2] : 0.0f;
    store16(orow + (size_t)w2 * ld + cvs * 8, v);
  }
}


// RGB fast path (Cc == 3, ld == 32): one thread per OUTPUT pixel, no shared memory.  The 12 (rt, rh, c) input rows are
// read as float2 (the two rw positions): a warp reads 256 contiguous bytes per row and writes 32 x 64 = 2 KB of
// contiguous output with four 16-byte stores per lane (a pure copy at HBM speed).
__global__ void __launch_bounds__(256) clip_to_s2d_rgb_kernel(const float* __restrict__ clip, int N, int T_, int H, int W,
                                                              __half* __restrict__ out) {
  const int T2 = T_ / 2, H2 = H / 2, W2 = W / 2;
  const long long total = (long long)N * T2 * H2 * W2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int w2 = (int)(idx % W2);
  long long r = idx / W2;
  const int h2 = (int)(r % H2); r /= H2;
  const int t2 = (int)(r % T2);
  const int n = (int)(r / T2);
  float v[32];
#pragma unroll
  for (int k = 24; k < 32; ++k) v[k] = 0.0f;
#pragma unroll
  for (int rt = 0; rt < 2; ++rt)
#pragma unroll
    for (int rh = 0; rh < 2; ++rh)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float2 p = __ldg(reinterpret_cast<const float2*>(
            clip + ((((size_t)n * T_ + 2 * t2 + rt) * 3 + c) * H + 2 * h2 + rh) * W + 2 * w2));
        const int q = (rt * 2 + rh) * 2;                 // channel ((rt*2+rh)*2+rw)*3 + c
        v[q * 3 + c] = p.x;
        v[(q + 1) * 3 + c] = p.y;
      }
  uint32_t o[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
    o[k] = *reinterpret_cast<const uint32_t*>(&h);
  }
  __half* dst = out + (size_t)idx * 32;
  uint4* d4 = reinterpret_cast<uint4*>(dst);   // 64 contiguous bytes as four 16-byte stores (sm_90 has no 32-byte stores)
#pragma unroll
  for (int k = 0; k < 4; ++k) d4[k] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
}

// [N*S, C] (ld) -> [N, C, S] fp32 via a 32x32 smem transpose
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ in, int S, int C, int ld, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z, s0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int s = s0 + i, c = c0 + threadIdx.x;
    if (s < S && c < C) tile[i][threadIdx.x] = to_f32<T>(in[((size_t)n * S + s) * ld + c]);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, s = s0 + threadIdx.x;
    if (s < S && c < C) out[((size_t)n * C + c) * S + s] = tile[threadIdx.x][i];
  }
}

template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, int S, int C, T* __restrict__ out, int ld) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z, s0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, s = s0 + threadIdx.x;
    if (s < S && c < C) tile[i][threadIdx.x] = in[((size_t)n * C + c) * S + s];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int s = s0 + i, c = c0 + threadIdx.x;
    if (s < S && c < C) out[((size_t)n * S + s) * ld + c] = from_f32<T>(tile[threadIdx.x][i]);
  }
}

// Small-N linear layers (global_cls N=60, local_reg / neighbor_reg N=4; K = 12544), split-K:
// CTA (kc, mt) stages an 8-row x KC-column tile of x in shared memory (fp32) and each warp sweeps
// output columns n = warp, warp+8, ...: lanes stream w[n, chunk] with 16-byte loads and multiply against
// the 8 staged rows.  Partials go to a [ksplit, M, N] workspace; linear_reduce_kernel sums them in a
// fixed order (deterministic), adds bias, optionally accumulates into y and applies the activation.
constexpr int kLinRows = 8;
constexpr int kLinKC = 512;
template <typename T>
__global__ void __launch_bounds__(256) linear_splitk_kernel(const T* __restrict__ x, int M, int K, int x_ld,
                                                            const T* __restrict__ w, int N,
                                                            const int32_t* __restrict__ row_map,
                                                            float* __restrict__ partial) {
  constexpr int VN = Vec16<T>::N;
  __shared__ __align__(16) float xs[kLinRows][kLinKC];
  const int kc = blockIdx.x, m0 = blockIdx.y * kLinRows;
  const int k0 = kc * kLinKC;
  const int klen = min(kLinKC, K - k0);  // multiple of VN
  for (int i = threadIdx.x; i < kLinRows * (kLinKC / VN); i += blockDim.x) {
    const int r = i / (kLinKC / VN), kv = i - r * (kLinKC / VN);
    float v[VN];
#pragma unroll
    for (int k = 0; k < VN; ++k) v[k] = 0.0f;
    if (m0 + r < M && kv * VN < klen) {
      const int xr = row_map ? row_map[m0 + r] : m0 + r;
      load16(x + (size_t)xr * x_ld + k0 + kv * VN, v);
    }
#pragma unroll
    for (int k = 0; k < VN; ++k) xs[r][kv * VN + k] = v[k];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int n = warp; n < N; n += nwarps) {
    float acc[kLinRows];
#pragma unroll
    for (int r = 0; r < kLinRows; ++r) acc[r] = 0.0f;
    const T* wr = w + (size_t)n * K + k0;
    for (int kv = lane; kv * VN < klen; kv += 32) {
      float wv[VN];
      load16(wr + kv * VN, wv);
#pragma unroll
      for (int r = 0; r < kLinRows; ++r) {
        const float4* xp = reinterpret_cast<const float4*>(&xs[r][kv * VN]);
#pragma unroll
        for (int q = 0; q < VN / 4; ++q) {
          float4 xv = xp[q];
          acc[r] = fmaf(xv.x, wv[4 * q + 0], acc[r]);
          acc[r] = fmaf(xv.y, wv[4 * q + 1], acc[r]);
          acc[r] = fmaf(xv.z, wv[4 * q + 2], acc[r]);
          acc[r] = fmaf(xv.w, wv[4 * q + 3], acc[r]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kLinRows; ++r) {
      float v = acc[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0 && m0 + r < M) partial[((size_t)kc * M + m0 + r) * N + n] = v;
    }
  }
}


// fp16 operands: the same split-K tiling on mma.sync tensor-core tiles, no shared memory.  One warp owns 16 rows and
// all N (<= 64) columns; per 32-column block every thread loads ONE 16-byte vector from each of its two rows of x and
// from one weight row per 8-column tile and feeds the four k-pairs it holds to two m16n8k16 steps.  The k order inside
// a block is therefore permuted (thread t covers columns 8t..8t+7), identically for x and w, which a dot product does
// not care about; x is streamed exactly once with full 32-byte sectors.
__device__ __forceinline__ void mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int NT>
__global__ void __launch_bounds__(128) linear_mma_kernel(const __half* __restrict__ x, int M, int K, int x_ld,
                                                         const __half* __restrict__ w, int N,
                                                         const int32_t* __restrict__ row_map, float* __restrict__ partial) {
  const int kc = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int m0 = blockIdx.y * 64 + warp * 16;
  if (m0 >= M) return;
  const int k0 = kc * kLinKC, klen = min(kLinKC, K - k0);   // multiple of 8
  const int r0 = m0 + g, r1 = m0 + g + 8;
  const bool v0 = r0 < M, v1 = r1 < M;
  const __half* xa = x + (size_t)(v0 ? (row_map ? row_map[r0] : r0) : 0) * x_ld + k0 + t * 8;
  const __half* xb = x + (size_t)(v1 ? (row_map ? row_map[r1] : r1) : 0) * x_ld + k0 + t * 8;
  const __half* wp[NT];
  bool wv[NT];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    wv[j] = j * 8 + g < N;
    wp[j] = w + (size_t)(wv[j] ? j * 8 + g : 0) * K + k0 + t * 8;
  }
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
  const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll 4
  for (int kb = 0; kb < klen; kb += 32) {
    const bool in = kb + t * 8 < klen;
    const uint4 a = (in && v0) ? *reinterpret_cast<const uint4*>(xa + kb) : zero;
    const uint4 b = (in && v1) ? *reinterpret_cast<const uint4*>(xb + kb) : zero;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const uint4 q = (in && wv[j]) ? *reinterpret_cast<const uint4*>(wp[j] + kb) : zero;
      mma_16816(acc[j], a.x, b.x, a.y, b.y, q.x, q.y);
      mma_16816(acc[j], a.z, b.z, a.w, b.w, q.z, q.w);
    }
  }
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int n = j * 8 + 2 * t;
    if (v0) {
      if (n < N) partial[((size_t)kc * M + r0) * N + n] = acc[j][0];
      if (n + 1 < N) partial[((size_t)kc * M + r0) * N + n + 1] = acc[j][1];
    }
    if (v1) {
      if (n < N) partial[((size_t)kc * M + r1) * N + n] = acc[j][2];
      if (n + 1 < N) partial[((size_t)kc * M + r1) * N + n + 1] = acc[j][3];
    }
  }
}

static void launch_linear_mma(const __half* x, int M, int K, int x_ld, const __half* w, int N, const int32_t* row_map,
                              float* partial, cudaStream_t s) {
  dim3 grid(ceil_div(K, kLinKC), ceil_div(M, 64));
  if (N <= 8) linear_mma_kernel<1><<<grid, 128, 0, s>>>(x, M, K, x_ld, w, N, row_map, partial);
  else if (N <= 16) linear_mma_kernel<2><<<grid, 128, 0, s>>>(x, M, K, x_ld, w, N, row_map, partial);
  else if (N <= 32) linear_mma_kernel<4><<<grid, 128, 0, s>>>(x, M, K, x_ld, w, N, row_map, partial);
  else linear_mma_kernel<8><<<grid, 128, 0, s>>>(x, M, K, x_ld, w, N, row_map, partial);
}

__global__ void linear_reduce_kernel(const float* __restrict__ partial, int ksplit, int M, int N,
                                     const float* __restrict__ bias, float* __restrict__ y, int y_ld, int act,
                                     int accumulate) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  int m = i / N, n = i - m * N;
  float v = 0.0f;
  for (int s = 0; s < ksplit; ++s) v += partial[((size_t)s * M + m) * N + n];
  v += bias ? bias[n] : 0.0f;
  float* dst = y + (size_t)m * y_ld + n;
  if (accumulate) v += *dst;
  if (act == 1) v = 1.0f / (1.0f + expf(-v));
  *dst = v;
}

// local_reg | neighbor_reg1 | neighbor_reg2 (two_branch.py:261-270) share their input: one split-K pass with the
// twelve weight rows, then this reduction writes local_loc [R,T,4], first_loc = (local + nb1)[:, s0:s1] and
// last_loc = (local + nb2)[:, e0:e1] in one go.  bias12 = [b_local | b_nb1 | b_nb2].
__global__ void head_reg_reduce_kernel(const float* __restrict__ partial, int ksplit, int R, int T,
                                       const float* __restrict__ bias12, int s0, int s1, int e0, int e1,
                                       float* __restrict__ local_loc, float* __restrict__ first, float* __restrict__ last) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (row m = r*T + t, coordinate c)
  const int M = R * T;
  if (i >= M * 4) return;
  const int m = i >> 2, c = i & 3;
  float v[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    float a = 0.0f;
    for (int s = 0; s < ksplit; ++s) a += partial[((size_t)s * M + m) * 12 + j * 4 + c];
    v[j] = a + bias12[j * 4 + c];
  }
  local_loc[i] = v[0];
  const int r = m / T, t = m - r * T;
  if (t >= s0 && t < s1) first[((size_t)r * (s1 - s0) + (t - s0)) * 4 + c] = v[0] + v[1];
  if (t >= e0 && t < e1) last[((size_t)r * (e1 - e0) + (t - e0)) * 4 + c] = v[0] + v[2];
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)kNumSMs * 16;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace step

using namespace step;

extern "C" int step_maxpool3d_fwd(const void* x, int dtype, int N, int T, int H, int W, int C, int in_ld, int KT,
                                  int KH, int KW, int ST, int SH, int SW, int PT, int PH, int PW, int pad_hi_t,
                                  int pad_hi_h, int pad_hi_w, int OT, int OH, int OW, void* y, int out_ld,
                                  step_stream_t stream) {
  const int vn = dtype == STEP_F16 ? 8 : 4;
  STEP_CHECK_ARG(dtype == STEP_F16 || dtype == STEP_F32, "maxpool3d: bad dtype");
  STEP_CHECK_ARG(x && y && N > 0 && T > 0 && H > 0 && W > 0, "maxpool3d: bad shape/pointer");
  STEP_CHECK_ARG(C % vn == 0 && in_ld % vn == 0 && out_ld % vn == 0, "maxpool3d: C/ld must be multiples of %d", vn);
  STEP_CHECK_ARG((((uintptr_t)x | (uintptr_t)y) & 15) == 0, "maxpool3d: pointers must be 16-byte aligned");
  if (KT == 3 && KH == 3 && KW == 3 && ST == 1 && SH == 1 && SW == 1 && PT == 1 && PH == 1 && PW == 1 && pad_hi_t == 1 &&
      pad_hi_h == 1 && pad_hi_w == 1 && OT == T && OH == H && OW == W && W % 7 == 0) {
    const long long per_seg = (long long)N * H * (W / 7) * (C / vn);
    int TS = T;
    while (TS > 2 && per_seg * ceil_div(T, TS) < 50000) TS = (TS + 1) / 2;
    const long long total = per_seg * ceil_div(T, TS);
    STEP_CHECK_ARG(ceil_div(total, 128) < (1LL << 31), "maxpool3d: too many blocks");
    if (dtype == STEP_F16)
      maxpool3d_333_march_kernel<__half><<<(unsigned)ceil_div(total, 128), 128, 0, cu(stream)>>>((const __half*)x, N, T, H, W, C,
                                                                                                 in_ld, (__half*)y, out_ld, TS);
    else
      maxpool3d_333_march_kernel<float><<<(unsigned)ceil_div(total, 128), 128, 0, cu(stream)>>>((const float*)x, N, T, H, W, C,
                                                                                                in_ld, (float*)y, out_ld, TS);
    STEP_LAUNCH_CHECK("maxpool3d_333_march_kernel");
    return 0;
  }
  {
    const bool k133 = KT == 1 && KH == 3 && KW == 3 && ST == 1 && SH == 2 && SW == 2;
    const bool k333 = KT == 3 && KH == 3 && KW == 3 && ST == 2 && SH == 2 && SW == 2;
    if (k133 || k333) {
      const int WB = k133 ? 7 : 4;
      const long long per_seg = (long long)N * OH * ceil_div(OW, WB) * (C / vn);
      int TS = k133 ? 1 : OT;
      while (TS > 2 && per_seg * ceil_div(OT, TS) < 50000) TS = (TS + 1) / 2;
      const long long total = per_seg * ceil_div(OT, TS);
      STEP_CHECK_ARG(ceil_div(total, 128) < (1LL << 31), "maxpool3d: too many blocks");
      const unsigned blocks = (unsigned)ceil_div(total, 128);
#define STEP_MARCH_GO(TT_, A, B, Cc, D, E, F, G)                                                                        \
      maxpool3d_march_kernel<TT_, A, B, Cc, D, E, F, G><<<blocks, 128, 0, cu(stream)>>>(                               \
          (const TT_*)x, N, T, H, W, C, in_ld, PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w, OT, OH, OW, (TT_*)y, out_ld, TS)
      if (dtype == STEP_F16) { if (k133) STEP_MARCH_GO(__half, 1, 3, 3, 1, 2, 2, 7); else STEP_MARCH_GO(__half, 3, 3, 3, 2, 2, 2, 4); }
      else { if (k133) STEP_MARCH_GO(float, 1, 3, 3, 1, 2, 2, 7); else STEP_MARCH_GO(float, 3, 3, 3, 2, 2, 2, 4); }
#undef STEP_MARCH_GO
      STEP_LAUNCH_CHECK("maxpool3d_march_kernel");
      return 0;
    }
  }
  // tile: up to 4 x 8 x 8 output pixels (whole rows on the small maps), 64-byte channel chunks
  const int TW = OW < 8 ? OW : (OW % 7 == 0 ? 7 : 8), TH = OH < 8 ? OH : (OH % 7 == 0 ? 7 : 8), TT = OT < 4 ? OT : 4;
  long long tiles = (long long)N * ceil_div(OT, TT) * ceil_div(OH, TH) * ceil_div(OW, TW);
  STEP_CHECK_ARG(tiles < (1LL << 31), "maxpool3d: too many tiles");
  const bool cv8 = (C / vn) % 8 == 0 && ((uintptr_t)x & 127) == 0 && (in_ld * (dtype == STEP_F16 ? 2 : 4)) % 128 == 0;
  dim3 grid((unsigned)tiles, ceil_div(C / vn, cv8 ? 8 : 4));
#define STEP_POOL_GO(TT_, A, B, Cc)                                                                                   \
  do {                                                                                                                \
    if (cv8)                                                                                                          \
      maxpool3d_kernel<TT_, A, B, Cc, 8><<<grid, 256, 0, cu(stream)>>>((const TT_*)x, N, T, H, W, C, in_ld, KT, KH, KW, ST, SH, \
                                                                      SW, PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w, OT, OH, \
                                                                      OW, (TT_*)y, out_ld, TT, TH, TW);               \
    else                                                                                                              \
      maxpool3d_kernel<TT_, A, B, Cc, 4><<<grid, 256, 0, cu(stream)>>>((const TT_*)x, N, T, H, W, C, in_ld, KT, KH, KW, ST, SH, \
                                                                      SW, PT, PH, PW, pad_hi_t, pad_hi_h, pad_hi_w, OT, OH, \
                                                                      OW, (TT_*)y, out_ld, TT, TH, TW);               \
  } while (0)
  const int kind = (KT == 1 && KH == 3 && KW == 3) ? 1 : ((KT == 3 && KH == 3 && KW == 3) ? 2 : 0);
  if (dtype == STEP_F16) {
    if (kind == 1) STEP_POOL_GO(__half, 1, 3, 3); else if (kind == 2) STEP_POOL_GO(__half, 3, 3, 3); else STEP_POOL_GO(__half, 0, 0, 0);
  } else {
    if (kind == 1) STEP_POOL_GO(float, 1, 3, 3); else if (kind == 2) STEP_POOL_GO(float, 3, 3, 3); else STEP_POOL_GO(float, 0, 0, 0);
  }
  (void)0;
#undef STEP_POOL_GO
  STEP_LAUNCH_CHECK("maxpool3d_kernel");
  return 0;
}

extern "C" int step_mean_mid_strided(const void* x, int dtype, int A, int B, int P, int C, int ld, long long a_stride, void* y,
                                     int out_dtype, step_stream_t stream) {
  STEP_CHECK_ARG(x && y && A > 0 && B > 0 && P > 0 && C > 0 && ld >= C, "mean_mid: bad args");
  STEP_CHECK_ARG(A == 1 || a_stride >= (long long)B * P * ld, "mean_mid: row stride %lld < B * P * ld", a_stride);
  long long total = (long long)A * P * C;
  int g = ceil_div(total, 256);
  if (dtype == STEP_F16 && C % 8 == 0 && ld % 8 == 0 && a_stride % 8 == 0 && ((uintptr_t)x & 15) == 0) {
    const int g8 = ceil_div(total / 8, 256);
    if (out_dtype == STEP_F16) mean_mid_h8_kernel<__half><<<g8, 256, 0, cu(stream)>>>((const __half*)x, A, B, P, C, ld, a_stride, (__half*)y);
    else if (out_dtype == STEP_F32) mean_mid_h8_kernel<float><<<g8, 256, 0, cu(stream)>>>((const __half*)x, A, B, P, C, ld, a_stride, (float*)y);
    else return fail(STEP_E_UNSUPPORTED, "mean_mid: dtype combination %d -> %d", dtype, out_dtype);
    STEP_LAUNCH_CHECK("mean_mid_h8_kernel");
    return 0;
  }
  if (dtype == STEP_F16 && out_dtype == STEP_F16)
    mean_mid_kernel<__half, __half><<<g, 256, 0, cu(stream)>>>((const __half*)x, A, B, P, C, ld, a_stride, (__half*)y);
  else if (dtype == STEP_F16 && out_dtype == STEP_F32)
    mean_mid_kernel<__half, float><<<g, 256, 0, cu(stream)>>>((const __half*)x, A, B, P, C, ld, a_stride, (float*)y);
  else if (dtype == STEP_F32 && out_dtype == STEP_F32)
    mean_mid_kernel<float, float><<<g, 256, 0, cu(stream)>>>((const float*)x, A, B, P, C, ld, a_stride, (float*)y);
  else
    return fail(STEP_E_UNSUPPORTED, "mean_mid: dtype combination %d -> %d", dtype, out_dtype);
  STEP_LAUNCH_CHECK("mean_mid_kernel");
  return 0;
}

extern "C" int step_mean_mid(const void* x, int dtype, int A, int B, int P, int C, int ld, void* y, int out_dtype,
                             step_stream_t stream) {
  return step_mean_mid_strided(x, dtype, A, B, P, C, ld, (long long)B * P * ld, y, out_dtype, stream);
}

extern "C" int step_clip_to_ndhwc(const float* clip, int N, int T, int Cc, int H, int W, void* out, int dtype, int ld,
                                  step_stream_t stream) {
  STEP_CHECK_ARG(clip && out && N > 0 && T > 0 && Cc > 0 && H > 0 && W > 0 && ld >= Cc, "clip_to_ndhwc: bad args");
  long long total = (long long)N * T * H * W;
  if (dtype == STEP_F16)
    clip_to_ndhwc_kernel<__half><<<grid_for(total, 256), 256, 0, cu(stream)>>>(clip, N, T, Cc, H, W, (__half*)out, ld);
  else if (dtype == STEP_F32)
    clip_to_ndhwc_kernel<float><<<grid_for(total, 256), 256, 0, cu(stream)>>>(clip, N, T, Cc, H, W, (float*)out, ld);
  else
    return fail(STEP_E_ARG, "clip_to_ndhwc: bad dtype");
  STEP_LAUNCH_CHECK("clip_to_ndhwc_kernel");
  return 0;
}

extern "C" int step_clip_to_s2d_f16(const float* clip, int N, int T, int Cc, int H, int W, void* out, int ld,
                                    step_stream_t stream) {
  STEP_CHECK_ARG(clip && out && N > 0 && T > 0 && Cc > 0 && H > 0 && W > 0, "clip_to_s2d: bad args");
  STEP_CHECK_ARG(T % 2 == 0 && H % 2 == 0 && W % 2 == 0 && ld >= 8 * Cc, "clip_to_s2d: T,H,W must be even, ld >= 8*Cc");
  STEP_CHECK_ARG(ld % 8 == 0 && ld <= 64 && 256 % (ld / 8) == 0 && (size_t)4 * Cc * W * sizeof(float) <= 48 * 1024, "clip_to_s2d: ld must divide 2048, row tile must fit 48 KB smem");
  STEP_CHECK_ARG(((uintptr_t)out & 15) == 0, "clip_to_s2d: out must be 16-byte aligned");
  if (Cc == 3 && ld == 32 && ((uintptr_t)clip & 7) == 0 && ((uintptr_t)out & 31) == 0) {
    const long long total = (long long)N * (T / 2) * (H / 2) * (W / 2);
    STEP_CHECK_ARG(ceil_div(total, 256) < (1LL << 31), "clip_to_s2d: too many pixels");
    clip_to_s2d_rgb_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, cu(stream)>>>(clip, N, T, H, W, (__half*)out);
    STEP_LAUNCH_CHECK("clip_to_s2d_rgb_kernel");
    return 0;
  }
  long long rows = (long long)N * (T / 2) * ceil_div(H / 2, kS2dRows);
  STEP_CHECK_ARG(rows < (1LL << 31), "clip_to_s2d: too many rows");
  clip_to_s2d_kernel<<<(unsigned)rows, 256, (size_t)4 * Cc * W * sizeof(float), cu(stream)>>>(clip, N, T, Cc, H, W, (__half*)out, ld);
  STEP_LAUNCH_CHECK("clip_to_s2d_kernel");
  return 0;
}

extern "C" int step_nhwc_to_nchw_f32(const void* in, int dtype, int N, int S, int C, int ld, float* out,
                                     step_stream_t stream) {
  STEP_CHECK_ARG(in && out && N > 0 && S > 0 && C > 0 && ld >= C && N <= 65535, "nhwc_to_nchw: bad args");
  dim3 grid(ceil_div(S, 32), ceil_div(C, 32), N), block(32, 8);
  if (dtype == STEP_F16)
    nhwc_to_nchw_kernel<__half><<<grid, block, 0, cu(stream)>>>((const __half*)in, S, C, ld, out);
  else if (dtype == STEP_F32)
    nhwc_to_nchw_kernel<float><<<grid, block, 0, cu(stream)>>>((const float*)in, S, C, ld, out);
  else
    return fail(STEP_E_ARG, "nhwc_to_nchw: bad dtype");
  STEP_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return 0;
}

extern "C" int step_nchw_to_nhwc(const float* in, int N, int S, int C, void* out, int dtype, int ld,
                                 step_stream_t stream) {
  STEP_CHECK_ARG(in && out && N > 0 && S > 0 && C > 0 && ld >= C && N <= 65535, "nchw_to_nhwc: bad args");
  dim3 grid(ceil_div(S, 32), ceil_div(C, 32), N), block(32, 8);
  if (dtype == STEP_F16)
    nchw_to_nhwc_kernel<__half><<<grid, block, 0, cu(stream)>>>(in, S, C, (__half*)out, ld);
  else if (dtype == STEP_F32)
    nchw_to_nhwc_kernel<float><<<grid, block, 0, cu(stream)>>>(in, S, C, (float*)out, ld);
  else
    return fail(STEP_E_ARG, "nchw_to_nhwc: bad dtype");
  STEP_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return 0;
}

extern "C" size_t step_linear_small_n_workspace_bytes(int M, int K, int N) {
  if (M <= 0 || K <= 0 || N <= 0) return 0;
  return (size_t)ceil_div(K, kLinKC) * M * N * sizeof(float);
}

extern "C" int step_linear_small_n(const void* x, int dtype, int M, int K, int x_ld, const void* w, const float* bias,
                                   int N, float* y, int y_ld, int act, int accumulate, const int32_t* row_map,
                                   void* workspace, size_t ws_bytes, step_stream_t stream) {
  const int vn = dtype == STEP_F16 ? 8 : 4;
  STEP_CHECK_ARG(dtype == STEP_F16 || dtype == STEP_F32, "linear_small_n: bad dtype");
  STEP_CHECK_ARG(x && w && y && M >= 0 && K > 0 && N > 0 && N <= 64 && y_ld >= N, "linear_small_n: bad args (N <= 64)");
  STEP_CHECK_ARG(K % vn == 0 && x_ld % vn == 0, "linear_small_n: K and x_ld must be multiples of %d", vn);
  STEP_CHECK_ARG((((uintptr_t)x | (uintptr_t)w) & 15) == 0, "linear_small_n: pointers must be 16-byte aligned");
  if (M == 0) return 0;
  const int ksplit = ceil_div(K, kLinKC);
  if (!workspace || ws_bytes < step_linear_small_n_workspace_bytes(M, K, N))
    return fail(STEP_E_WORKSPACE, "linear_small_n: workspace %zu < %zu", ws_bytes, step_linear_small_n_workspace_bytes(M, K, N));
  dim3 grid(ksplit, ceil_div(M, kLinRows));
  STEP_CHECK_ARG(grid.y <= 65535, "linear_small_n: M too large");
  const int threads = N >= 8 ? 256 : 32 * N;
  if (dtype == STEP_F16)
    launch_linear_mma((const __half*)x, M, K, x_ld, (const __half*)w, N, row_map, (float*)workspace, cu(stream));
  else
    linear_splitk_kernel<float><<<grid, threads, 0, cu(stream)>>>((const float*)x, M, K, x_ld, (const float*)w, N,
                                                                   row_map, (float*)workspace);
  STEP_LAUNCH_CHECK("linear_splitk_kernel");
  linear_reduce_kernel<<<ceil_div((long long)M * N, 256), 256, 0, cu(stream)>>>((const float*)workspace, ksplit, M, N, bias,
                                                                               y, y_ld, act, accumulate);
  STEP_LAUNCH_CHECK("linear_reduce_kernel");
  return 0;
}

extern "C" int step_head_regress(const void* x, int dtype, int R, int T, int K, int x_ld, const void* w12,
                                 const float* bias12, int s0, int s1, int e0, int e1, float* local_loc, float* first,
                                 float* last, void* workspace, size_t ws_bytes, step_stream_t stream) {
  const int vn = dtype == STEP_F16 ? 8 : 4;
  const int M = R * T;
  STEP_CHECK_ARG(dtype == STEP_F16 || dtype == STEP_F32, "head_regress: bad dtype");
  STEP_CHECK_ARG(x && w12 && bias12 && local_loc && first && last && R >= 0 && T > 0 && K > 0, "head_regress: bad args");
  STEP_CHECK_ARG(0 <= s0 && s0 < s1 && s1 <= T && 0 <= e0 && e0 < e1 && e1 <= T, "head_regress: bad chunk ranges");
  STEP_CHECK_ARG(K % vn == 0 && x_ld % vn == 0 && (((uintptr_t)x | (uintptr_t)w12) & 15) == 0, "head_regress: alignment");
  if (M == 0) return 0;
  const int ksplit = ceil_div(K, kLinKC);
  if (!workspace || ws_bytes < step_linear_small_n_workspace_bytes(M, K, 12))
    return fail(STEP_E_WORKSPACE, "head_regress: workspace %zu < %zu", ws_bytes, step_linear_small_n_workspace_bytes(M, K, 12));
  dim3 grid(ksplit, ceil_div(M, kLinRows));
  STEP_CHECK_ARG(grid.y <= 65535, "head_regress: too many rows");
  if (dtype == STEP_F16)
    launch_linear_mma((const __half*)x, M, K, x_ld, (const __half*)w12, 12, nullptr, (float*)workspace, cu(stream));
  else
    linear_splitk_kernel<float><<<grid, 256, 0, cu(stream)>>>((const float*)x, M, K, x_ld, (const float*)w12, 12, nullptr,
                                                              (float*)workspace);
  STEP_LAUNCH_CHECK("linear_splitk_kernel");
  head_reg_reduce_kernel<<<ceil_div((long long)M * 4, 256), 256, 0, cu(stream)>>>((const float*)workspace, ksplit, R, T, bias12,
                                                                                 s0, s1, e0, e1, local_loc, first, last);
  STEP_LAUNCH_CHECK("head_reg_reduce_kernel");
  return 0;
}
