// dropout.cuh -- the keep decision of torch.nn.functional.dropout on a CUDA tensor (ATen's fused_dropout_kernel_vec), as a
// function of the draw's generator state and the element's index in the tensor torch drops.  It is the only place that
// knows how torch lays its Philox stream over the elements; every dropout kernel of train.cu asks it, in the forward and,
// regenerating the mask from (seed, offset) instead of storing it, in the backward.
//
// torch launches 256-thread blocks, grid = min(ceil(n / 256), multiProcessorCount * (maxThreadsPerMultiProcessor / 256)),
// n_threads = 256 * grid.  On a 16-byte aligned contiguous fp32 tensor with n % 4 == 0, thread idx runs
// curand_init(seed, idx, offset), and its j-th curand_uniform4 covers the elements 4 * (idx + n_threads * j) ... + 3, one
// component each; an element is kept iff its uniform is < (float)(1 - p).  Kept values are
// x * (float)(1.0 / (double)(float)(1 - p)).  The generator's offset then advances by ((n - 1) / (n_threads * 4) + 1) * 4.
// Measured against torch 2.11 on an H100 (tests/test_gpu_dropout.py), including the seed's high word and offsets that
// start past zero.
#pragma once
#include <curand_philox4x32_x.h>

namespace step {

struct DropDraw {
  unsigned long long seed, offset;
  float keep, scale;           // (float)(1 - p), (float)(1.0 / (double)keep)
  unsigned int n_threads;      // torch's 256 * grid
};

// Index of an element of the dropped tensor from its coordinates in the caller's layout: base + r*s_r + t*s_t + p*s_p + c*s_c.
struct DropMap {
  long long base, s_r;
  int s_t, s_p, s_c;
  __device__ __forceinline__ long long at(long long r, int t, int p, int c) const {
    return base + r * s_r + (long long)t * s_t + (long long)p * s_p + (long long)c * s_c;
  }
};

// true iff element e of the draw is kept.  curand_uniform4's k-th call on a state made by curand_init(seed, idx, offset)
// returns the words (offset & 3) + 4k ... + 3 of the stream Philox4x32-10(counter = offset / 4 + w / 4, subsequence idx),
// word w % 4 of each block; its uniform is word * 2^-32 + 2^-33 (the product is exact, so contraction cannot change it).
__device__ __forceinline__ bool drop_keep(const DropDraw& d, long long e) {
  const long long v = e >> 2;
  const unsigned int idx = (unsigned int)(v % d.n_threads);
  const unsigned long long k = (unsigned long long)(v / d.n_threads);
  const unsigned long long w = (d.offset & 3ULL) + 4ULL * k + (unsigned long long)(e & 3);
  const unsigned long long ctr = (d.offset >> 2) + (w >> 2);
  const uint4 r = curand_Philox4x32_10(make_uint4((unsigned int)ctr, (unsigned int)(ctr >> 32), idx, 0u),
                                       make_uint2((unsigned int)d.seed, (unsigned int)(d.seed >> 32)));
  const int q = (int)(w & 3ULL);
  const unsigned int x = q == 0 ? r.x : q == 1 ? r.y : q == 2 ? r.z : r.w;
  const float u = __fadd_rn(__fmul_rn(__uint2float_rn(x), 2.3283064365386963e-10f), 1.1641532182693481e-10f);
  return u < d.keep;
}

// the factor an element of the draw is multiplied by: scale if kept, else 0
__device__ __forceinline__ float drop_factor(const DropDraw& d, long long e) { return drop_keep(d, e) ? d.scale : 0.0f; }

}  // namespace step
