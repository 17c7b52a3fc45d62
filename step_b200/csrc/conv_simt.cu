// conv_simt.cu -- channels-last 3-D convolution on CUDA cores (fp32 accumulate), the precision
// reference path: cfg.fp16 == False runs it in fp32 storage (parity with the reference's fp32
// Conv3d/Conv2d/BatchNorm3d, models/i3dpt.py:103-111, two_branch.py:60-111); the same kernel with
// __half storage cross-checks the tensor-core kernel (conv_umma.cu) on identical inputs.
//
// Implicit GEMM, CTA tile 64 pixels x 64 output channels, K step 16 input channels per filter tap,
// 4x4 register micro-tile per thread, zero-fill for the TF-"SAME" halo (i3dpt.py:14-31).
// Epilogue: y = relu?( acc * scale[c] + shift[c] + residual ).
#include "common.cuh"

namespace step {

constexpr int BM = 64, BN = 64, BK = 16;

template <typename T>
__global__ void __launch_bounds__(256) conv3d_simt_kernel(step_conv_params p) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const T* __restrict__ x = (const T*)p.x;
  const T* __restrict__ w = (const T*)p.w;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 4 (pixels) x 4 (channels)
  const long long M = (long long)p.N * p.OT * p.OH * p.OW;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // loader roles: A: pixel lp = tid / 4, channel quad lq = tid % 4;  B: cout = tid / 4, quad = tid % 4
  const int lp = tid >> 2, lq = tid & 3;
  long long am = m0 + lp;
  const bool a_valid = am < M;
  int a_n = 0, a_t = 0, a_h = 0, a_w = 0;
  if (a_valid) {
    a_w = (int)(am % p.OW); long long r = am / p.OW;
    a_h = (int)(r % p.OH); r /= p.OH;
    a_t = (int)(r % p.OT); a_n = (int)(r / p.OT);
  }
  const int b_co = n0 + lp;
  const bool b_valid = b_co < p.Cout;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  const int taps = p.KT * p.KH * p.KW;
  for (int tap = 0; tap < taps; ++tap) {
    const int kw = tap % p.KW, kh = (tap / p.KW) % p.KH, kt = tap / (p.KW * p.KH);
    const int it = a_t * p.ST + kt - p.PT, ih = a_h * p.SH + kh - p.PH, iw = a_w * p.SW + kw - p.PW;
    const bool in_ok = a_valid && it >= 0 && it < p.T && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
    const T* xa = x + ((((size_t)a_n * p.T + it) * p.H + ih) * p.W + iw) * p.in_ld;
    const T* wb = w + ((size_t)b_co * taps + tap) * p.w_ld;
    for (int c0 = 0; c0 < p.Cin; c0 += BK) {
      const int c = c0 + lq * 4;
      float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4] = {0.f, 0.f, 0.f, 0.f};
      if (in_ok && c < p.Cin) {
#pragma unroll
        for (int k = 0; k < 4; ++k) av[k] = to_f32<T>(xa[c + k]);
      }
      if (b_valid && c < p.Cin) {
#pragma unroll
        for (int k = 0; k < 4; ++k) bv[k] = to_f32<T>(wb[c + k]);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 4; ++k) { As[lq * 4 + k][lp] = av[k]; Bs[lq * 4 + k][lp] = bv[k]; }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; b[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
  }

  T* __restrict__ y = (T*)p.y;
  const T* __restrict__ res = (const T*)p.residual;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = n0 + tx * 4 + j;
      if (co >= p.Cout) continue;
      float v = acc[i][j];
      if (p.scale) v *= p.scale[co];
      if (p.shift) v += p.shift[co];
      if (res) v += to_f32<T>(res[(size_t)m * p.res_ld + p.res_coff + co]);
      if (p.relu) v = fmaxf(v, 0.0f);
      y[(size_t)m * p.out_ld + p.out_coff + co] = from_f32<T>(v);
    }
  }
}

int conv3d_simt_launch(const step_conv_params* p, step_stream_t stream) {
  STEP_CHECK_ARG(p->Cin % 4 == 0 && p->w_ld >= p->Cin && p->in_ld >= p->Cin,
                 "conv3d(simt): Cin=%d must be a multiple of 4 (pad), w_ld=%d in_ld=%d", p->Cin, p->w_ld, p->in_ld);
  long long M = (long long)p->N * p->OT * p->OH * p->OW;
  dim3 grid(ceil_div(M, BM), ceil_div(p->Cout, BN));
  if (p->dtype == STEP_F16)
    conv3d_simt_kernel<__half><<<grid, 256, 0, cu(stream)>>>(*p);
  else
    conv3d_simt_kernel<float><<<grid, 256, 0, cu(stream)>>>(*p);
  STEP_LAUNCH_CHECK("conv3d_simt_kernel");
  return 0;
}

}  // namespace step
