// bottleneck_exit.cu -- the exit of one 2-D bottleneck of the local branch fused with the 1x1 convolution that consumes it
// (reference: models/two_branch.py:60-84 Bottleneck.forward `out = conv3(out); out += residual; out = relu(out)`, :86-111
// Bottleneck_resample.forward, followed by the next block's `conv1` + ReLU (:68-69) or by `downsample2` (:259)):
//
//     Y[M, 1024] = relu(H[M, 256] * W3[1024, 256]^T + X[M, 1024])          conv3 + residual + ReLU     (stored unless y == NULL)
//     Z[M,  256] = act(Y[M, 1024] * W1[256, 1024]^T + shift2)               next conv1 (ReLU) / downsample2 (bias, no ReLU)
//
// As two launches of the implicit-GEMM kernel the 1024-wide Y makes a round trip through HBM between them.  Here a CTA owns
// 64 rows and walks the 1024 columns of Y in 16 chunks of 64: consumer warpgroup (chunk & 1) computes the GEMM1 chunk with
// wgmma (registers), adds the residual, applies the ReLU, rounds to fp16 and writes the chunk as a K-major 128B-swizzled A
// operand into shared memory (and to Y when it is stored); then both warpgroups accumulate Z += Y_chunk * W1[:, chunk]^T, each
// for 128 of Z's 256 columns.  Y is rounded to fp16 before GEMM2 exactly as the two-launch path rounds it, and both GEMMs issue
// the same m64n64k16 wgmma sequence in the same K order as conv_umma.cu, so the results are bit-identical to the unfused path.
//
// Per CTA (384 threads): warp 0 loads H and the W3 chunks (TMA, 3-slot ring), warp 1 loads the W1 slices (2-slot ring),
// warpgroups 1 and 2 compute.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "common.cuh"
#include "umma_ptx.cuh"

namespace step {
namespace bexit {

constexpr int kThreads = 384;
constexpr int BM = 64;                          // rows per CTA
constexpr int K1 = 256, N1 = 1024, N2 = 256, CH = 64, NCH = N1 / CH;   // 16 chunks of 64 columns of Y
constexpr int kHBytes = 4 * BM * 128;           // H tile: 4 k-blocks x [64 rows x 128 B]
constexpr int kW3Bytes = 4 * CH * 128;          // W3 chunk: 4 k-blocks x [64 rows x 128 B]
constexpr int kW1Bytes = N2 * 128;              // W1 slice: [256 rows x 128 B]
constexpr int kYBytes = BM * 128;               // Y chunk: [64 rows x 128 B]
constexpr int kW3Ring = 3, kW1Ring = 2;

struct Geom {
  int M, store_y, relu2, x_ld, y_ld, z_ld;
};

struct Bars {
  uint64_t h_full;
  uint64_t w3_full[kW3Ring], w3_empty[kW3Ring];
  uint64_t w1_full[kW1Ring], w1_empty[kW1Ring];
};

__global__ void __launch_bounds__(kThreads, 1)
bottleneck_exit_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w3,
                       const __grid_constant__ CUtensorMap map_w1, Geom g, const float* __restrict__ shift2,
                       const __half* __restrict__ x, __half* __restrict__ y, __half* __restrict__ z) {
  extern __shared__ __align__(1024) uint8_t raw[];
  Bars* bars = (Bars*)raw;
  uint8_t* base = (uint8_t*)(((uintptr_t)raw + sizeof(Bars) + 1023) & ~(uintptr_t)1023);
  uint8_t* sH = base;
  uint8_t* sW3 = sH + kHBytes;
  uint8_t* sW1 = sW3 + kW3Ring * kW3Bytes;
  uint8_t* sY = sW1 + kW1Ring * kW1Bytes;        // [2][kYBytes]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_h) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w3) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w1) : "memory");
    mbar_init(&bars->h_full, 1);
    for (int i = 0; i < kW3Ring; ++i) { mbar_init(&bars->w3_full[i], 1); mbar_init(&bars->w3_empty[i], 1); }
    for (int i = 0; i < kW1Ring; ++i) { mbar_init(&bars->w1_full[i], 1); mbar_init(&bars->w1_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  if (warp == 0) {
    if (elect_one()) {
      mbar_expect_tx(&bars->h_full, kHBytes);
      for (int kb = 0; kb < 4; ++kb) tma_load_2d(&map_h, &bars->h_full, sH + kb * BM * 128, kb * 64, m0);
      for (int c = 0; c < NCH; ++c) {
        const int s = c % kW3Ring;
        mbar_wait(&bars->w3_empty[s], ((uint32_t)(c / kW3Ring) & 1u) ^ 1u);
        mbar_expect_tx(&bars->w3_full[s], kW3Bytes);
        for (int kb = 0; kb < 4; ++kb)
          tma_load_2d(&map_w3, &bars->w3_full[s], sW3 + s * kW3Bytes + kb * CH * 128, kb * 64, c * CH);
      }
    }
  } else if (warp == 1) {
    if (elect_one()) {
      for (int c = 0; c < NCH; ++c) {
        const int s = c % kW1Ring;
        mbar_wait(&bars->w1_empty[s], ((uint32_t)(c / kW1Ring) & 1u) ^ 1u);
        mbar_expect_tx(&bars->w1_full[s], kW1Bytes);
        tma_load_2d(&map_w1, &bars->w1_full[s], sW1 + s * kW1Bytes, c * CH, 0);
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp >> 2) - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint64_t hi = desc_hi_kmajor<64>();
    const uint64_t h_lo = desc_lo(sH), w3_lo = desc_lo(sW3), w1_lo = desc_lo(sW1), y_lo = desc_lo(sY);
    const int r0 = (warp & 3) * 16 + (lane >> 2);          // rows r0, r0 + 8 of the tile
    float accz[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) accz[i] = 0.0f;
    mbar_wait(&bars->h_full, 0);
    for (int p = 0; p < NCH / 2; ++p) {
      // ---- GEMM1: this warpgroup's chunk c1 of Y ----
      const int c1 = 2 * p + wg, s3 = c1 % kW3Ring;
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
      mbar_wait(&bars->w3_full[s3], (uint32_t)(c1 / kW3Ring) & 1u);
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_64x64(acc, hi | (h_lo + (uint64_t)((kb * BM * 128) >> 4) + 2 * k),
                      hi | (w3_lo + (uint64_t)((s3 * kW3Bytes + kb * CH * 128) >> 4) + 2 * k), 1u);
      wg_commit();
      wg_wait<0>();
      if (leader) mbar_arrive(&bars->w3_empty[s3]);
      // ---- residual + ReLU -> fp16 Y chunk (swizzled A operand; Y in global memory when stored) ----
      uint8_t* ybuf = sY + wg * kYBytes;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = r0 + 8 * i;
        const bool valid = m0 + r < g.M;
        const __half* xrow = x + (size_t)(m0 + r) * g.x_ld + c1 * CH;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          float f0 = fmaf(acc[4 * j + 2 * i], 1.0f, 0.0f), f1 = fmaf(acc[4 * j + 2 * i + 1], 1.0f, 0.0f);
          if (valid) {
            const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(xrow + col));
            f0 += rf.x; f1 += rf.y;
          }
          f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f);
          const __half2 hv = __floats2half2_rn(f0, f1);
          *reinterpret_cast<__half2*>(ybuf + r * 128 + ((j ^ (r & 7)) << 4) + 4 * (lane & 3)) = hv;
          if (valid && g.store_y) *reinterpret_cast<__half2*>(y + (size_t)(m0 + r) * g.y_ld + c1 * CH + col) = hv;
        }
      }
      fence_proxy_async();                                  // generic-proxy writes of Y -> visible to wgmma
      named_sync(1, 256);
      // ---- GEMM2: Z[:, 128 wg + (0..127)] += Y_chunk(c) * W1[:, chunk c]^T for c = 2p, 2p + 1, in K order ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = 2 * p + h, s1 = c % kW1Ring;
        mbar_wait(&bars->w1_full[s1], (uint32_t)(c / kW1Ring) & 1u);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int n = 0; n < 2; ++n)
            wgmma_64x64(accz + n * 32, hi | (y_lo + (uint64_t)((h * kYBytes) >> 4) + 2 * k),
                        hi | (w1_lo + (uint64_t)((s1 * kW1Bytes + (128 * wg + 64 * n) * 128) >> 4) + 2 * k), 1u);
        wg_commit();
      }
      wg_wait<0>();
      if (leader) { mbar_arrive(&bars->w1_empty[0]); mbar_arrive(&bars->w1_empty[1]); }
      named_sync(1, 256);                                   // both Y buffers are free for the next pair
    }
    // ---- Z epilogue: + shift2, optional ReLU, fp16 ----
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + 8 * i;
      if (m0 + r >= g.M) continue;
      __half* zrow = z + (size_t)(m0 + r) * g.z_ld + 128 * wg;
#pragma unroll
      for (int n = 0; n < 2; ++n)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = 64 * n + 8 * j + 2 * (lane & 3);
          const float b0 = shift2 ? shift2[128 * wg + col] : 0.0f, b1 = shift2 ? shift2[128 * wg + col + 1] : 0.0f;
          float f0 = fmaf(accz[n * 32 + 4 * j + 2 * i], 1.0f, b0), f1 = fmaf(accz[n * 32 + 4 * j + 2 * i + 1], 1.0f, b1);
          if (g.relu2) { f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f); }
          *reinterpret_cast<__half2*>(zrow + col) = __floats2half2_rn(f0, f1);
        }
    }
  }
}

typedef CUresult (*EncFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                          const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncFn g_enc = nullptr;

// [rows, cols] fp16, row pitch ld elements; box [box_r rows x 64 columns] = 128-byte rows, 128B swizzle
static int enc2d(CUtensorMap* m, const void* base, int cols, long long rows, long long ld, int box_r, CUtensorMapL2promotion pr) {
  cuuint64_t d[2] = {(cuuint64_t)cols, (cuuint64_t)rows}, st[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_r}, es[2] = {1, 1};
  CUresult r = g_enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), d, st, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, pr, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

}  // namespace bexit
}  // namespace step

extern "C" int step_bottleneck_exit_f16(const void* h, long long h_ld, const void* w3, const void* x, long long x_ld, const void* w1,
                                        const float* shift2, int relu2, void* y, long long y_ld, void* z, long long z_ld,
                                        long long M, int planes, int inplanes, int outplanes, step_stream_t stream) {
  using namespace step;
  using namespace step::bexit;
  STEP_CHECK_ARG(h && w3 && x && w1 && z, "bottleneck_exit: null pointer");
  STEP_CHECK_ARG(planes == K1 && inplanes == N1 && outplanes == N2,
                 "bottleneck_exit: built for planes 256, inplanes 1024, outplanes 256 (two_branch.py:190-192), got %d / %d / %d",
                 planes, inplanes, outplanes);
  STEP_CHECK_ARG(M >= 1 && M <= 0x7fffff00LL, "bottleneck_exit: M = %lld", M);
  STEP_CHECK_ARG(h_ld >= K1 && x_ld >= N1 && z_ld >= N2 && (!y || y_ld >= N1), "bottleneck_exit: row pitch below the channel count");
  STEP_CHECK_ARG(h_ld % 8 == 0 && x_ld % 8 == 0 && z_ld % 8 == 0 && (!y || y_ld % 8 == 0), "bottleneck_exit: row pitches must keep 16-byte alignment");
  STEP_CHECK_ARG(((uintptr_t)h | (uintptr_t)w3 | (uintptr_t)w1 | (uintptr_t)y | (uintptr_t)x | (uintptr_t)z) % 16 == 0,
                 "bottleneck_exit: pointers must be 16-byte aligned");
  if (!g_enc) {
    cudaDriverEntryPointQueryResult q;
    void* f = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || !f)
      return fail(STEP_E_DRIVER, "cuTensorMapEncodeTiled entry point unavailable");
    g_enc = (EncFn)f;
  }
  CUtensorMap mh, mw3, mw1;
  int r;
  if ((r = enc2d(&mh, h, K1, M, h_ld, BM, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return fail(STEP_E_DRIVER, "bottleneck_exit: tensor map h (%d)", r);
  if ((r = enc2d(&mw3, w3, K1, N1, K1, CH, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return fail(STEP_E_DRIVER, "bottleneck_exit: tensor map w3 (%d)", r);
  if ((r = enc2d(&mw1, w1, N1, N2, N1, N2, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return fail(STEP_E_DRIVER, "bottleneck_exit: tensor map w1 (%d)", r);
  Geom g;
  g.M = (int)M; g.store_y = y ? 1 : 0; g.relu2 = relu2 ? 1 : 0; g.x_ld = (int)x_ld; g.y_ld = (int)y_ld; g.z_ld = (int)z_ld;
  const size_t smem = sizeof(Bars) + 1024 + kHBytes + kW3Ring * kW3Bytes + kW1Ring * kW1Bytes + 2 * kYBytes;
  static std::atomic<unsigned long long> attr_seen{0};
  if (first_use_on_device(attr_seen)) {
    cudaError_t e = cudaFuncSetAttribute(bottleneck_exit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail((int)e, "bottleneck_exit: smem attribute: %s", cudaGetErrorString(e));
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  cfg.gridDim = dim3((unsigned)((M + BM - 1) / BM));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = cu(stream);
  cudaError_t le = cudaLaunchKernelEx(&cfg, bottleneck_exit_kernel, mh, mw3, mw1, g, shift2, (const __half*)x, (__half*)y, (__half*)z);
  if (le != cudaSuccess) { cudaGetLastError(); return fail((int)le, "bottleneck_exit_kernel launch: %s", cudaGetErrorString(le)); }
  STEP_LAUNCH_CHECK("bottleneck_exit_kernel");
  return 0;
}
