// bottleneck_exit.cu -- the exit of one 2-D bottleneck of the local branch fused with the 1x1 convolution that consumes it
// (reference: models/two_branch.py:60-84 Bottleneck.forward `out = conv3(out); out += residual; out = relu(out)`, :86-111
// Bottleneck_resample.forward, followed by the next block's `conv1` + ReLU (:68-69) or by `downsample2` (:259)):
//
//     Y[M, 1024] = relu(H[M, 256] * W3[1024, 256]^T + X[M, 1024])          conv3 + residual + ReLU     (stored unless y == NULL)
//     Z[M,  256] = act(Y[M, 1024] * W1[256, 1024]^T + shift2)               next conv1 (ReLU) / downsample2 (bias, no ReLU)
//
// As two launches of the implicit-GEMM kernel the 1024-wide Y makes a round trip through HBM between them.  Here a CTA owns
// 128 rows; consumer warpgroup wg owns rows [64 wg, 64 wg + 64) and walks the 1024 columns of Y in 16 chunks of 64:
//   GEMM1   acc[64 x 64] = H * W3[chunk]^T                    16 x m64n64k16, both operands in shared memory
//   epilogue acc + residual (X chunk, TMA-loaded), ReLU, fp16 -> written back over the X chunk for the TMA store of Y, and
//           kept in registers: accumulator registers [8 kk, 8 kk + 8) are the A fragment of k-step kk of GEMM2
//   GEMM2   Z[64 x 256] += Y_chunk * W1[:, chunk]^T            4 x m64n256k16, A in registers, Z in 128 registers
// GEMM1 of chunk c + 1 is issued right behind GEMM2 of chunk c.  The two consumer warpgroups share the weight rings and no
// other barrier (a staggered start and a 2-CTA weight multicast were measured and did not pay, DESIGN.md section 3.1).
// Y is rounded to fp16 before GEMM2 exactly as the two-launch path rounds it, and both GEMMs accumulate K in ascending
// 16-wide steps as conv_umma.cu does, so the results are bit-identical to the unfused path.  Z is staged in the warpgroup's (then finished) rows of the H tile and stored by TMA;
// the tensor maps clip the ragged last tile.
//
// Per CTA (384 threads): warp 0 loads H and the W3 chunks, warp 1 the W1 slices, warps 2 and 3 the X chunks of consumer
// warpgroup 0 and 1 (TMA, one thread per ring, two slots each); warpgroups 1 and 2 compute, with the producer warpgroup's
// registers handed to them (setmaxnreg 40 / 232).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "common.cuh"
#include "umma_ptx.cuh"

namespace step {
namespace bexit {

constexpr int kThreads = 384;
constexpr int BM = 128;                         // rows per CTA, 64 per consumer warpgroup
constexpr int K1 = 256, N1 = 1024, N2 = 256, CH = 64, NCH = N1 / CH;   // 16 chunks of 64 columns of Y
constexpr int kHBytes = 4 * BM * 128;           // H tile: 4 k-blocks x [128 rows x 128 B]
constexpr int kW3Bytes = 4 * CH * 128;          // W3 chunk: 4 k-blocks x [64 rows x 128 B]
constexpr int kW1Bytes = N2 * 128;              // W1 slice: [256 rows x 128 B]
constexpr int kXBytes = 64 * 128;               // one warpgroup's X / Y chunk: [64 rows x 128 B]
constexpr int kRing = 2;                        // slots of every ring
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

struct Geom {
  int M, store_y, relu2;
};

struct Bars {
  uint64_t h_full;
  uint64_t w3_full[kRing], w3_empty[kRing];
  uint64_t w1_full[kRing], w1_empty[kRing];
  uint64_t x_full[2][kRing], x_empty[2][kRing];   // per consumer warpgroup
};

__global__ void __launch_bounds__(kThreads, 1)
bottleneck_exit_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w3,
                       const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_x,
                       const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_z, Geom g,
                       const float* __restrict__ shift2) {
  extern __shared__ __align__(1024) uint8_t raw[];
  Bars* bars = (Bars*)raw;
  uint8_t* base = (uint8_t*)(((uintptr_t)raw + sizeof(Bars) + 1023) & ~(uintptr_t)1023);
  uint8_t* sH = base;
  uint8_t* sW3 = sH + kHBytes;
  uint8_t* sW1 = sW3 + kRing * kW3Bytes;
  uint8_t* sX = sW1 + kRing * kW1Bytes;          // [slot][warpgroup][kXBytes]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_h);
    prefetch_tensormap(&map_w3);
    prefetch_tensormap(&map_w1);
    prefetch_tensormap(&map_x);
    if (g.store_y) prefetch_tensormap(&map_y);
    prefetch_tensormap(&map_z);
    mbar_init(&bars->h_full, 1);
    for (int i = 0; i < kRing; ++i) {
      mbar_init(&bars->w3_full[i], 1); mbar_init(&bars->w3_empty[i], 2);
      mbar_init(&bars->w1_full[i], 1); mbar_init(&bars->w1_empty[i], 2);
      for (int w = 0; w < 2; ++w) { mbar_init(&bars->x_full[w][i], 1); mbar_init(&bars->x_empty[w][i], 1); }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      if (elect_one()) {
        mbar_expect_tx(&bars->h_full, kHBytes);
        for (int kb = 0; kb < 4; ++kb) tma_load_2d(&map_h, &bars->h_full, sH + kb * BM * 128, kb * 64, m0);
        for (int c = 0; c < NCH; ++c) {
          const int s = c % kRing;
          mbar_wait(&bars->w3_empty[s], ((uint32_t)(c / kRing) & 1u) ^ 1u);
          mbar_expect_tx(&bars->w3_full[s], kW3Bytes);
          for (int kb = 0; kb < 4; ++kb)
            tma_load_2d(&map_w3, &bars->w3_full[s], sW3 + s * kW3Bytes + kb * CH * 128, kb * 64, c * CH);
        }
      }
    } else if (warp == 1) {
      if (elect_one()) {
        for (int c = 0; c < NCH; ++c) {
          const int s = c % kRing;
          mbar_wait(&bars->w1_empty[s], ((uint32_t)(c / kRing) & 1u) ^ 1u);
          mbar_expect_tx(&bars->w1_full[s], kW1Bytes);
          tma_load_2d(&map_w1, &bars->w1_full[s], sW1 + s * kW1Bytes, c * CH, 0);
        }
      }
    } else {
      const int wg = warp - 2;
      if (m0 + 64 * wg < g.M && elect_one()) {    // the last tile's second warpgroup may have no rows: no X to load
        for (int c = 0; c < NCH; ++c) {
          const int s = c % kRing;
          mbar_wait(&bars->x_empty[wg][s], ((uint32_t)(c / kRing) & 1u) ^ 1u);
          mbar_expect_tx(&bars->x_full[wg][s], kXBytes);
          tma_load_2d(&map_x, &bars->x_full[wg][s], sX + (s * 2 + wg) * kXBytes, c * CH, m0 + 64 * wg);
        }
      }
    }
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    if (m0 + 64 * wg >= g.M) {
      // No rows (the second half of a last tile of at most 64 rows): release every weight slot in the order the other
      // warpgroup does, and compute nothing.  Waiting for each slot to fill first keeps these arrivals in the slot's
      // current phase: the next fill of a slot needs the other warpgroup's release of it too.
      if (leader)
        for (int c = 0; c < NCH; ++c) {
          const int s = c % kRing;
          const uint32_t ph = (uint32_t)(c / kRing) & 1u;
          mbar_wait(&bars->w3_full[s], ph);
          mbar_arrive(&bars->w3_empty[s]);
          mbar_wait(&bars->w1_full[s], ph);
          mbar_arrive(&bars->w1_empty[s]);
        }
      return;
    }
    const uint64_t hi = desc_hi_kmajor<64>();
    const uint64_t h_lo = desc_lo(sH + wg * 64 * 128), w3_lo = desc_lo(sW3), w1_lo = desc_lo(sW1);
    const int r0 = (warp & 3) * 16 + (lane >> 2);          // rows r0, r0 + 8 of the warpgroup's 64
    const int t4 = 4 * (lane & 3);                          // byte offset of the thread's column pair in a 16-byte chunk
    float accz[128], acc[32];
#pragma unroll
    for (int i = 0; i < 128; ++i) accz[i] = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
    // GEMM1 of chunk c into acc: W3 chunk c sits in slot c % kRing
    auto gemm1 = [&](int c) {
      const int s3 = c % kRing;
      mbar_wait(&bars->w3_full[s3], (uint32_t)(c / kRing) & 1u);
      wg_fence();
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_f16<64>(acc, hi | (h_lo + (uint64_t)((kb * BM * 128) >> 4) + 2 * k),
                        hi | (w3_lo + (uint64_t)((s3 * kW3Bytes + kb * CH * 128) >> 4) + 2 * k), 1u);
      wg_commit();
    };
    mbar_wait(&bars->h_full, 0);
    gemm1(0);
    wg_wait<0>();
    if (leader) mbar_arrive(&bars->w3_empty[0]);
    for (int c = 0; c < NCH; ++c) {
      const int s = c % kRing;
      const uint32_t ph = (uint32_t)(c / kRing) & 1u;
      uint8_t* xb = sX + (s * 2 + wg) * kXBytes;
      // ---- residual + ReLU -> fp16 Y chunk: GEMM2's A fragments, and over the X chunk for the store ----
      uint32_t a[16];
      mbar_wait(&bars->x_full[wg][s], ph);
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = r0 + 8 * i;
          __half2* px = reinterpret_cast<__half2*>(xb + r * 128 + ((j ^ (r & 7)) << 4) + t4);
          float f0 = fmaf(acc[4 * j + 2 * i], 1.0f, 0.0f), f1 = fmaf(acc[4 * j + 2 * i + 1], 1.0f, 0.0f);
          const float2 rf = __half22float2(*px);
          f0 += rf.x; f1 += rf.y;
          f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f);
          const __half2 hv = __floats2half2_rn(f0, f1);
          if (g.store_y) *px = hv;
          a[4 * (j >> 1) + 2 * (j & 1) + i] = *reinterpret_cast<const uint32_t*>(&hv);
        }
      if (g.store_y) fence_proxy_async();                 // generic-proxy writes of Y -> visible to the TMA store
      named_sync(1 + wg, 128);                            // the whole warpgroup is done with the X chunk
      if (leader) {
        if (g.store_y) { tma_store_2d(&map_y, xb, c * CH, m0 + 64 * wg); bulk_commit(); }
        else mbar_arrive(&bars->x_empty[wg][s]);
      }
      // ---- GEMM2: Z += Y_chunk(c) * W1[:, chunk c]^T, then GEMM1 of the next chunk behind it ----
      mbar_wait(&bars->w1_full[s], ph);
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_f16_ra<256>(accz, a + 4 * kk, hi | (w1_lo + (uint64_t)((s * kW1Bytes) >> 4) + 2 * kk), 1u);
      wg_commit();
      if (c + 1 < NCH) {
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
        gemm1(c + 1);
      }
      if (leader && g.store_y) { bulk_wait_read<0>(); mbar_arrive(&bars->x_empty[wg][s]); }
      wg_wait<0>();
      if (leader) {
        mbar_arrive(&bars->w1_empty[s]);
        if (c + 1 < NCH) mbar_arrive(&bars->w3_empty[(c + 1) % kRing]);
      }
    }
    // ---- Z epilogue: + shift2, optional ReLU, fp16, staged as 4 column blocks of 64 in this warpgroup's rows of H ----
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      uint8_t* zb = sH + n * BM * 128 + wg * 64 * 128;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = 64 * n + 8 * j + (t4 >> 1);
        const float b0 = shift2 ? shift2[col] : 0.0f, b1 = shift2 ? shift2[col + 1] : 0.0f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = r0 + 8 * i;
          float f0 = fmaf(accz[4 * (8 * n + j) + 2 * i], 1.0f, b0), f1 = fmaf(accz[4 * (8 * n + j) + 2 * i + 1], 1.0f, b1);
          if (g.relu2) { f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f); }
          *reinterpret_cast<__half2*>(zb + r * 128 + ((j ^ (r & 7)) << 4) + t4) = __floats2half2_rn(f0, f1);
        }
      }
    }
    fence_proxy_async();
    named_sync(1 + wg, 128);
    if (leader) {
      for (int n = 0; n < 4; ++n) tma_store_2d(&map_z, sH + n * BM * 128 + wg * 64 * 128, 64 * n, m0 + 64 * wg);
      bulk_commit();
      bulk_wait_read<0>();
    }
  }
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
  CUtensorMap mh, mw3, mw1, mx, my, mz;
  memset(&my, 0, sizeof(my));
  // row matrices in boxes of 64 columns = 128-byte rows, 128B swizzle
  const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
  const CUtensorMapL2promotion act = CU_TENSOR_MAP_L2_PROMOTION_L2_128B, wgt = CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
  int rc;
  if ((rc = encode_rows2d(&mh, h, M, K1, h_ld, 64, BM, sw, act, "bottleneck_exit: h")) ||
      (rc = encode_rows2d(&mw3, w3, N1, K1, K1, 64, CH, sw, wgt, "bottleneck_exit: w3")) ||
      (rc = encode_rows2d(&mw1, w1, N2, N1, N1, 64, N2, sw, wgt, "bottleneck_exit: w1")) ||
      (rc = encode_rows2d(&mx, x, M, N1, x_ld, 64, 64, sw, act, "bottleneck_exit: x")) ||
      (y && (rc = encode_rows2d(&my, y, M, N1, y_ld, 64, 64, sw, act, "bottleneck_exit: y"))) ||
      (rc = encode_rows2d(&mz, z, M, N2, z_ld, 64, 64, sw, act, "bottleneck_exit: z")))
    return rc;
  Geom g;
  g.M = (int)M; g.store_y = y ? 1 : 0; g.relu2 = relu2 ? 1 : 0;
  const size_t smem = sizeof(Bars) + 1024 + kHBytes + kRing * (kW3Bytes + kW1Bytes + 2 * kXBytes);
  static std::atomic<unsigned long long> attr_seen{0};
  if ((rc = allow_dynamic_smem(bottleneck_exit_kernel, attr_seen, (int)smem, "bottleneck_exit_kernel"))) return rc;
  return launch_tc("bottleneck_exit_kernel", bottleneck_exit_kernel, dim3((unsigned)((M + BM - 1) / BM)), kThreads, smem,
                   cu(stream), mh, mw3, mw1, mx, my, mz, g, shift2);
}
