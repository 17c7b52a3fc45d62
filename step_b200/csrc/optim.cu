// optim.cu -- the parameter update of the training step (train.py:123-128, 345-348 of the reference) as multi-tensor
// launches over a device table of step_optim_tensor rows and a block -> (tensor, chunk) map:
//   * nonfinite_kernel  one pass over every gradient; stores 1 to a device flag if any element is inf or NaN (the skip
//                       test of dynamic loss scaling, apex O1 at train.py:136-137, 342-345);
//   * adam_kernel       torch.optim.Adam (amsgrad=False, maximize=False, L2 weight decay added to the gradient);
//   * sgd_kernel        torch.optim.SGD (dampening=0, nesterov=False).
// One CTA updates one chunk of one tensor; elements are independent, so there are no atomics and no reductions.
// Each tensor whose pointers are all 16-byte aligned takes 16-byte vector loads and stores; unaligned tensors and the ragged
// end of a chunk take the scalar path.
//
// Rounding: this file is compiled with -fmad=false and spells every operation with an explicitly rounded intrinsic in the
// order of the torch kernels the single-tensor torch optimizers launch one after another: `a + alpha * x` (add, lerp,
// addcmul with x = b * c, addcdiv with x = b / c) is one fused multiply-add inside its torch kernel, while the separate kernels of
// `(v.sqrt() / bc2_sqrt).add_(eps)` each round (torch divides by a host scalar as a multiply by its reciprocal, which it
// takes in double and rounds to float: the host passes that reciprocal).
// Without -fmad=false the compiler could contract the latter across what torch rounds separately.
#include "common.cuh"

namespace step {

constexpr int kOptThreads = 256;
constexpr long long kOptChunk = 16384;            // elements per CTA (16 float4 per thread), step_multi_tensor_chunk()
static_assert(kOptChunk % (4 * kOptThreads) == 0, "a chunk is whole float4 per thread");

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__global__ void __launch_bounds__(kOptThreads) nonfinite_kernel(const step_optim_tensor* __restrict__ table, int n_tensors,
                                                                const step_optim_block* __restrict__ blocks,
                                                                int* __restrict__ flag) {
  const step_optim_block b = blocks[blockIdx.x];
  if (b.tensor < 0 || b.tensor >= n_tensors) return;
  const float* __restrict__ g = table[b.tensor].grad;
  const long long start = (long long)b.chunk * kOptChunk;
  const long long n = min(kOptChunk, table[b.tensor].numel - start);
  bool bad = false;
  long long nvec = 0;
  if (n > 0 && aligned16(g)) {
    nvec = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g + start);
    for (long long i = threadIdx.x; i < nvec; i += kOptThreads) {
      const float4 v = g4[i];
      bad |= !isfinite(v.x) | !isfinite(v.y) | !isfinite(v.z) | !isfinite(v.w);
    }
    nvec <<= 2;
  }
  for (long long i = nvec + threadIdx.x; i < n; i += kOptThreads) bad |= !isfinite(g[start + i]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) *flag = 1;
}

struct AdamScalars {
  float neg_step_size, inv_bc2_sqrt, wd, w1, beta2, w2, eps;
};

// torch.optim.Adam, _single_tensor_adam, one element:
//   grad = grad.add(param, alpha=wd); exp_avg.lerp_(grad, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
//   denom = (exp_avg_sq.sqrt() / bc2_sqrt).add_(eps); param.addcdiv_(exp_avg, denom, value=-step_size)
__device__ __forceinline__ void adam_elem(const AdamScalars& s, float& p, float g, float& m, float& v) {
  if (s.wd != 0.0f) g = __fmaf_rn(s.wd, p, g);
  const float d = __fsub_rn(g, m);
  m = s.w1 < 0.5f ? __fmaf_rn(s.w1, d, m) : __fmaf_rn(-d, __fsub_rn(1.0f, s.w1), g);    // ATen lerp, both branches
  v = __fmaf_rn(s.w2, __fmul_rn(g, g), __fmul_rn(v, s.beta2));                            // ATen addcmul: a + alpha * (b * c)
  const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(v), s.inv_bc2_sqrt), s.eps);
  p = __fmaf_rn(s.neg_step_size, __fdiv_rn(m, denom), p);
}

__global__ void __launch_bounds__(kOptThreads) adam_kernel(const step_optim_tensor* __restrict__ table, int n_tensors,
                                                           const step_optim_block* __restrict__ blocks) {
  const step_optim_block b = blocks[blockIdx.x];
  if (b.tensor < 0 || b.tensor >= n_tensors) return;
  const step_optim_tensor& t = table[b.tensor];
  const long long start = (long long)b.chunk * kOptChunk;
  const long long n = min(kOptChunk, t.numel - start);
  if (n <= 0) return;
  AdamScalars s;
  s.neg_step_size = -t.step_size;
  s.inv_bc2_sqrt = t.inv_bias_correction2_sqrt;
  s.wd = t.weight_decay; s.w1 = t.one_minus_beta1; s.beta2 = t.beta2; s.w2 = t.one_minus_beta2; s.eps = t.eps;
  float* __restrict__ p = t.param + start;
  const float* __restrict__ g = t.grad + start;
  float* __restrict__ m = t.exp_avg + start;
  float* __restrict__ v = t.exp_avg_sq + start;
  long long nvec = 0;
  if (aligned16(t.param) && aligned16(t.grad) && aligned16(t.exp_avg) && aligned16(t.exp_avg_sq)) {
    nvec = n >> 2;
    for (long long i = threadIdx.x; i < nvec; i += kOptThreads) {
      float4 p4 = reinterpret_cast<float4*>(p)[i], m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
      const float4 g4 = reinterpret_cast<const float4*>(g)[i];
      adam_elem(s, p4.x, g4.x, m4.x, v4.x);
      adam_elem(s, p4.y, g4.y, m4.y, v4.y);
      adam_elem(s, p4.z, g4.z, m4.z, v4.z);
      adam_elem(s, p4.w, g4.w, m4.w, v4.w);
      reinterpret_cast<float4*>(p)[i] = p4; reinterpret_cast<float4*>(m)[i] = m4; reinterpret_cast<float4*>(v)[i] = v4;
    }
    nvec <<= 2;
  }
  for (long long i = nvec + threadIdx.x; i < n; i += kOptThreads) {
    float pe = p[i], me = m[i], ve = v[i];
    adam_elem(s, pe, g[i], me, ve);
    p[i] = pe; m[i] = me; v[i] = ve;
  }
}

// torch.optim.SGD, _single_tensor_sgd, one element:
//   grad = grad.add(param, alpha=wd); buf = grad.clone() on the first step, else buf.mul_(momentum).add_(grad);
//   param.add_(buf, alpha=-lr)   (no buffer when momentum == 0)
__device__ __forceinline__ void sgd_elem(float neg_lr, float wd, float mom, int init, float& p, float g, float* buf) {
  if (wd != 0.0f) g = __fmaf_rn(wd, p, g);
  if (buf) {
    g = init ? g : __fadd_rn(__fmul_rn(*buf, mom), g);
    *buf = g;
  }
  p = __fmaf_rn(neg_lr, g, p);
}

__global__ void __launch_bounds__(kOptThreads) sgd_kernel(const step_optim_tensor* __restrict__ table, int n_tensors,
                                                          const step_optim_block* __restrict__ blocks) {
  const step_optim_block b = blocks[blockIdx.x];
  if (b.tensor < 0 || b.tensor >= n_tensors) return;
  const step_optim_tensor& t = table[b.tensor];
  const long long start = (long long)b.chunk * kOptChunk;
  const long long n = min(kOptChunk, t.numel - start);
  if (n <= 0) return;
  const float neg_lr = -t.step_size, wd = t.weight_decay, mom = t.momentum;
  const int init = t.buf_uninit;
  float* __restrict__ p = t.param + start;
  const float* __restrict__ g = t.grad + start;
  float* __restrict__ m = t.exp_avg ? t.exp_avg + start : nullptr;
  long long nvec = 0;
  if (aligned16(t.param) && aligned16(t.grad) && aligned16(t.exp_avg)) {
    nvec = n >> 2;
    for (long long i = threadIdx.x; i < nvec; i += kOptThreads) {
      float4 p4 = reinterpret_cast<float4*>(p)[i];
      const float4 g4 = reinterpret_cast<const float4*>(g)[i];
      float4 m4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m && !init) m4 = reinterpret_cast<float4*>(m)[i];
      sgd_elem(neg_lr, wd, mom, init, p4.x, g4.x, m ? &m4.x : nullptr);
      sgd_elem(neg_lr, wd, mom, init, p4.y, g4.y, m ? &m4.y : nullptr);
      sgd_elem(neg_lr, wd, mom, init, p4.z, g4.z, m ? &m4.z : nullptr);
      sgd_elem(neg_lr, wd, mom, init, p4.w, g4.w, m ? &m4.w : nullptr);
      reinterpret_cast<float4*>(p)[i] = p4;
      if (m) reinterpret_cast<float4*>(m)[i] = m4;
    }
    nvec <<= 2;
  }
  for (long long i = nvec + threadIdx.x; i < n; i += kOptThreads) {
    float pe = p[i], me = 0.0f;
    if (m && !init) me = m[i];
    sgd_elem(neg_lr, wd, mom, init, pe, g[i], m ? &me : nullptr);
    p[i] = pe;
    if (m) m[i] = me;
  }
}

static int check_table(const char* name, const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks,
                       int n_blocks) {
  STEP_CHECK_ARG(n_tensors >= 0 && n_blocks >= 0, "%s: negative count (n_tensors %d, n_blocks %d)", name, n_tensors, n_blocks);
  STEP_CHECK_ARG(n_tensors > 0 || (table == nullptr && n_blocks == 0 && blocks == nullptr),
                 "%s: n_tensors == 0 with a non-null table, block map or n_blocks %d", name, n_blocks);
  STEP_CHECK_ARG(n_tensors == 0 || table != nullptr, "%s: null pointer (table) for %d tensors", name, n_tensors);
  STEP_CHECK_ARG(n_blocks == 0 || blocks != nullptr, "%s: null pointer (block map) for %d blocks", name, n_blocks);
  return 0;
}

}  // namespace step

extern "C" int step_multi_tensor_chunk(void) { return (int)step::kOptChunk; }

extern "C" int step_multi_tensor_nonfinite_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks,
                                               int n_blocks, int* flag, step_stream_t stream) {
  using namespace step;
  if (int rc = check_table("step_multi_tensor_nonfinite_f32", table, n_tensors, blocks, n_blocks)) return rc;
  STEP_CHECK_ARG(flag != nullptr, "step_multi_tensor_nonfinite_f32: null pointer (flag)");
  cudaError_t e = cudaMemsetAsync(flag, 0, sizeof(int), cu(stream));
  if (e != cudaSuccess) return fail((int)e, "step_multi_tensor_nonfinite_f32: clearing the flag: %s", cudaGetErrorString(e));
  if (n_blocks == 0) return 0;
  nonfinite_kernel<<<n_blocks, kOptThreads, 0, cu(stream)>>>(table, n_tensors, blocks, flag);
  STEP_LAUNCH_CHECK("nonfinite_kernel");
  return 0;
}

extern "C" int step_multi_tensor_adam_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks,
                                          int n_blocks, step_stream_t stream) {
  using namespace step;
  if (int rc = check_table("step_multi_tensor_adam_f32", table, n_tensors, blocks, n_blocks)) return rc;
  if (n_blocks == 0) return 0;
  adam_kernel<<<n_blocks, kOptThreads, 0, cu(stream)>>>(table, n_tensors, blocks);
  STEP_LAUNCH_CHECK("adam_kernel");
  return 0;
}

extern "C" int step_multi_tensor_sgd_f32(const step_optim_tensor* table, int n_tensors, const step_optim_block* blocks,
                                         int n_blocks, step_stream_t stream) {
  using namespace step;
  if (int rc = check_table("step_multi_tensor_sgd_f32", table, n_tensors, blocks, n_blocks)) return rc;
  if (n_blocks == 0) return 0;
  sgd_kernel<<<n_blocks, kOptThreads, 0, cu(stream)>>>(table, n_tensors, blocks);
  STEP_LAUNCH_CHECK("sgd_kernel");
  return 0;
}
