// common.cuh -- shared host/device helpers for libstep_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/step_b200.h"

namespace step {

// thread-local last error text (step_last_error)
char* err_buf();
void count_launch();
int fail(int code, const char* fmt, ...);

inline cudaStream_t cu(step_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

#define STEP_CHECK_ARG(cond, ...)                              \
  do {                                                         \
    if (!(cond)) return step::fail(STEP_E_ARG, __VA_ARGS__);   \
  } while (0)

// after every launch: count it and surface launch-configuration errors without synchronising
#define STEP_LAUNCH_CHECK(name)                                                     \
  do {                                                                              \
    step::count_launch();                                                           \
    cudaError_t e__ = cudaPeekAtLastError();                                        \
    if (e__ != cudaSuccess) {                                                       \
      cudaGetLastError();                                                           \
      return step::fail((int)e__, "%s: %s", name, cudaGetErrorString(e__));        \
    }                                                                               \
  } while (0)

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

constexpr int kNumSMs = 132;  // H100 SXM

// The ROIPool backward (train.cu) accumulates one frame's [H*W, chunk] fp32 tile in shared memory, chunk >= 8 channels:
// maps of up to 6400 pixels (80x80, inputs up to ~1280x1280).  The argmax forward (roi.cu) checks the same limit, so a
// training step fails before its forward rather than after it.
constexpr int kPoolBwdSmem = 200 * 1024;
constexpr int kPoolBwdMinChunk = 8;
constexpr int kPoolBwdMaxPixels = kPoolBwdSmem / (kPoolBwdMinChunk * (int)sizeof(float));

// Function attributes (dynamic shared memory limit) are per device: a process driving several GPUs (nn.DataParallel,
// test.py:79-95 of the reference) must set them once on each.  `seen` is a per-kernel bitmask owned by the caller.
inline bool first_use_on_device(std::atomic<unsigned long long>& seen) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ULL << (dev & 63);
  return (seen.fetch_or(bit, std::memory_order_relaxed) & bit) == 0;
}

// Raise `kernel`'s dynamic shared-memory limit to `bytes`, once per device (`seen` as above).
template <typename Kernel>
inline int allow_dynamic_smem(Kernel kernel, std::atomic<unsigned long long>& seen, int bytes, const char* label) {
  if (!first_use_on_device(seen)) return 0;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return fail((int)e, "%s: shared memory attribute: %s", label, cudaGetErrorString(e));
  return 0;
}

// ---- device helpers -----------------------------------------------------------------------
template <typename T>
struct Vec16;  // 16-byte vector of T
template <>
struct Vec16<float> {
  static constexpr int N = 4;
  float v[4];
};
template <>
struct Vec16<__half> {
  static constexpr int N = 8;
  __half v[8];
};

template <typename T>
__device__ __forceinline__ float to_f32(T x);
template <>
__device__ __forceinline__ float to_f32<float>(float x) { return x; }
template <>
__device__ __forceinline__ float to_f32<__half>(__half x) { return __half2float(x); }

template <typename T>
__device__ __forceinline__ T from_f32(float x);
template <>
__device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }

template <typename T>
__device__ __forceinline__ void load16(const T* p, float* out) {
  uint4 raw = *reinterpret_cast<const uint4*>(p);
  if constexpr (sizeof(T) == 4) {
    out[0] = __uint_as_float(raw.x); out[1] = __uint_as_float(raw.y);
    out[2] = __uint_as_float(raw.z); out[3] = __uint_as_float(raw.w);
  } else {
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __half22float2(h[i]);
      out[2 * i] = f.x; out[2 * i + 1] = f.y;
    }
  }
}

template <typename T>
__device__ __forceinline__ void store16(T* p, const float* in) {
  uint4 raw;
  if constexpr (sizeof(T) == 4) {
    raw.x = __float_as_uint(in[0]); raw.y = __float_as_uint(in[1]);
    raw.z = __float_as_uint(in[2]); raw.w = __float_as_uint(in[3]);
  } else {
    __half2* h = reinterpret_cast<__half2*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(in[2 * i], in[2 * i + 1]);
  }
  *reinterpret_cast<uint4*>(p) = raw;
}

}  // namespace step
