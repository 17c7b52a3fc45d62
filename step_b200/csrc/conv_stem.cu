// conv_stem.cu -- the space-to-depth I3D stem (models/i3dpt.py:184-190 as engine.pack_stem_s2d packs it: a 4x4x4 stride-1
// filter, pad 1, 64 output channels, over the s2d clip [N, T/2, H/2, W/2, ld >= 24] whose 24 live channels are RGB x 2x2x2).
//
// The generic patch kernel (conv_halo.cu) puts pixels on the wgmma M side and the 64 output channels on N, so every MMA is
// m64n64k16 with both operands read from shared memory (4 KB per 64 K-steps of tensor work: the SM's shared-memory rate
// with no slack), and it multiplies the 8 padding channels of the 32-channel s2d layout.  Here the GEMM is transposed:
//   D^T[64 Cout, pixels] = W[64, K] * X^T[K, pixels],
// weights are A (M = the 64 output channels, one warpgroup covers all of them) and one 16 h x 8 w output plane is
// B (N = 128 pixels).  A CTA owns 4 planes x 16 x 8 pixels; consumer warpgroup wg computes planes 2 wg and 2 wg + 1.
//
// K holds only the 3 live 8-channel groups.  A k16 step pairs the same channel group g at two vertically neighbouring taps
// (kh, kw) and (kh + 1, kw) through the descriptors' K-direction stride (LBO): one patch row on the pixel side, four weight
// blocks on the weight side.  For the last t tap plane (k_t = 6, 7) the rt = 1 channels 12..23 carry zero weights
// (engine.pack_stem_s2d, zero_cin_last_kt in include/step_b200.h), so its channel-group-2 steps are not issued: 88 k16
// steps per plane instead of 128 in the 32-channel problem.
//
// Shared memory (no swizzle, wgmma K-major core matrices of 8 rows x 16 bytes):
//   patch  [3 channel groups][7 t][19 h][11 w][8 channels], one TMA box per group, zero fill outside the clip = the halo;
//          B core matrices are 8 consecutive w pixels, SBO = LBO = one patch row.
//   ring   stages of two filter rows (kt, kh..kh+1) = 8 taps: [group][tap][64 Cout][8 channels], one TMA box (1 KB) per
//          (group, tap); A core matrices are 8 output channels, SBO = 128 bytes, LBO = 4 blocks.
// Epilogue: folded BN scale / shift per accumulator row (= output channel) + ReLU, fp16, transposed by stmatrix into a
// pixel-major staging tile in the ring, then 16-byte coalesced stores of the channels-last output.
//
// Warp roles (384 threads): warp 0 producer (patch + weight ring), warpgroups 1 and 2 consumers.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "umma_ptx.cuh"

namespace step {

constexpr int kStemThreads = 384;
constexpr int kStemTT = 4, kStemTH = 16, kStemTW = 8;                      // output tile: 4 planes of 16 x 8 pixels
constexpr int kStemGroups = 3;                                             // live 8-channel groups
constexpr int kStemHpT = kStemTT + 3, kStemHpH = kStemTH + 3, kStemHpW = kStemTW + 3;   // patch of a 4x4x4 filter
constexpr int kStemPlanePix = kStemHpH * kStemHpW;
constexpr int kStemChunk = (kStemHpT * kStemPlanePix * 16 + 127) / 128 * 128;   // one channel group, TMA-aligned
constexpr int kStemBlock = 64 * 16;                                        // 64 output channels x 8 input channels
constexpr int kStemStageBytes = kStemGroups * 8 * kStemBlock;              // 8 taps
constexpr int kStemStages = 6;
constexpr int kStemSteps = 8;                                              // stages per CTA: 4 kt x 2 kh pairs
constexpr int kStemBook = 1024;                                            // barriers
constexpr int kStemPitch = 144;                                            // staging row: 64 fp16 + 16 bytes (banks)
constexpr int kStemSmem = kStemBook + 1024 + kStemStages * kStemStageBytes + kStemGroups * kStemChunk;
static_assert(kStemSmem <= 227 * 1024, "stem kernel exceeds shared memory");
static_assert(kStemTT * kStemTH * kStemTW * kStemPitch <= kStemStages * kStemStageBytes, "staging tile exceeds the ring");
// descriptor high words: [16,30) LBO >> 4, [32,46) SBO >> 4, no swizzle
constexpr uint64_t kStemAHi = ((uint64_t)((4 * kStemBlock) >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
constexpr uint64_t kStemBHi = ((uint64_t)((kStemHpW * 16) >> 4) << 16) | ((uint64_t)((kStemHpW * 16) >> 4) << 32);

struct StemGeom {
  int OT, OH, OW, tiles_w, tiles_h, tiles_t;
  int out_ld, out_coff, relu;
};

// One weight stage (filter rows kt, kh0 and kh0 + 1) for the warpgroup's two planes: NG channel groups x 4 kw k16 steps.
// a_lo: the stage in the ring; b_lo: the patch pixel of tap (kt, kh0, 0) for the warpgroup's first plane (16-byte units).
template <int NG>
__device__ __forceinline__ void stem_mma_stage(float (&acc)[2][64], uint64_t a_lo, uint64_t b_lo) {
#pragma unroll
  for (int kw = 0; kw < 4; ++kw)
#pragma unroll
    for (int gi = 0; gi < NG; ++gi)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        wgmma_f16<128>(acc[j], kStemAHi | (a_lo + (uint64_t)((gi * 8 + kw) * (kStemBlock >> 4))),
                       kStemBHi | (b_lo + (uint64_t)(gi * (kStemChunk >> 4) + j * kStemPlanePix + kw)), 1u);
}

template <int NG>
__device__ __forceinline__ void stem_stage(float (&acc)[2][64], int st, int wg, bool leader, uint8_t* ring, uint8_t* patch,
                                           uint64_t* full_bar, uint64_t* empty_bar) {
  const int s = st % kStemStages;
  mbar_wait(&full_bar[s], (uint32_t)(st / kStemStages) & 1u);
  const int kt = st >> 1, kh0 = (st & 1) * 2;
  const uint64_t a_lo = desc_lo(ring + (size_t)s * kStemStageBytes);
  const uint64_t b_lo = desc_lo(patch) + (uint64_t)((2 * wg + kt) * kStemPlanePix + kh0 * kStemHpW);
  wg_fence();
  stem_mma_stage<NG>(acc, a_lo, b_lo);
  wg_commit();
  wg_wait<1>();                                  // the previous stage's MMAs have retired: free it
  if (st > 0 && leader) mbar_arrive(&empty_bar[(st - 1) % kStemStages]);
}

__global__ void __launch_bounds__(kStemThreads, 1)
conv_stem_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, StemGeom g,
                 const float* __restrict__ scale, const float* __restrict__ shift, __half* __restrict__ y) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint64_t* full_bar = (uint64_t*)smem_raw;            // [kStemStages] weight stage landed
  uint64_t* empty_bar = full_bar + kStemStages;        // [kStemStages] weight stage consumed by both warpgroups
  uint64_t* pfull_bar = empty_bar + kStemStages;       // patch landed
  uint8_t* ring = (uint8_t*)(((uintptr_t)smem_raw + kStemBook + 1023) & ~(uintptr_t)1023);
  uint8_t* patch = ring + kStemStages * kStemStageBytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int b = blockIdx.x;
  const int tw = b % g.tiles_w; b /= g.tiles_w;
  const int th = b % g.tiles_h; b /= g.tiles_h;
  const int tt = b % g.tiles_t;
  const int n = b / g.tiles_t;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    prefetch_tensormap(&map_w);
    for (int s = 0; s < kStemStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_init(pfull_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== producer =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      mbar_expect_tx(pfull_bar, (uint32_t)(kStemGroups * kStemHpT * kStemPlanePix * 16));
      for (int c = 0; c < kStemGroups; ++c)
        tma_load_5d(&map_x, pfull_bar, patch + (size_t)c * kStemChunk, c * 8, tw * kStemTW - 1, th * kStemTH - 1,
                    tt * kStemTT - 1, n);
      for (int st = 0; st < kStemSteps; ++st) {
        const int s = st % kStemStages, use = st / kStemStages;
        if (use > 0) mbar_wait(&empty_bar[s], (uint32_t)(use - 1) & 1u);
        const int ng = st < kStemSteps - 2 ? kStemGroups : kStemGroups - 1;   // last t tap plane: group 2 is zero
        mbar_expect_tx(&full_bar[s], (uint32_t)(ng * 8 * kStemBlock));
        uint8_t* dst = ring + (size_t)s * kStemStageBytes;
        for (int c = 0; c < ng; ++c)
          for (int j = 0; j < 8; ++j)
            tma_load_3d(&map_w, &full_bar[s], dst + (c * 8 + j) * kStemBlock, c * 8, st * 8 + j, 0);
      }
    }
  } else {
    // ===================== consumers =====================
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;                      // planes 2 wg, 2 wg + 1 of the tile
    const int ct = threadIdx.x - 128;
    const bool leader = ct % 128 == 0;
    float acc[2][64];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[j][i] = 0.0f;
    mbar_wait(pfull_bar, 0);
    // the stage split is compile-time: a data-dependent guard around the wgmma issue would make ptxas serialise it
    for (int st = 0; st < kStemSteps - 2; ++st) stem_stage<kStemGroups>(acc, st, wg, leader, ring, patch, full_bar, empty_bar);
    for (int st = kStemSteps - 2; st < kStemSteps; ++st)
      stem_stage<kStemGroups - 1>(acc, st, wg, leader, ring, patch, full_bar, empty_bar);
    wg_wait<0>();
    // accumulator rows (output channels) of this thread: co and co + 8; columns 8 q + 2 (lane % 4) + {0, 1} = h q, w
    const int co = (warp & 3) * 16 + (lane >> 2);
    float sc[2], sh[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      sc[i] = scale ? scale[co + 8 * i] : 1.0f;
      sh[i] = shift ? shift[co + 8 * i] : 0.0f;
    }
    // both warpgroups are done with the ring and the patch: the ring becomes the [512 pixels][64 channels] staging tile
    named_sync(1, 256);
    const int m = lane >> 3;                             // stmatrix: matrix m = (h row q + m / 2, channels + 8 (m % 2))
    const uint32_t lane_addr = smem_u32(ring) + (uint32_t)(((m >> 1) * 8 + (lane & 7)) * kStemPitch +
                                                           ((warp & 3) * 16 + (m & 1) * 8) * 2);
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 16; q += 2) {
        uint32_t v[4];
#pragma unroll
        for (int mm = 0; mm < 4; ++mm) {
          const int qq = q + (mm >> 1), i = mm & 1;
          float f0 = fmaf(acc[j][4 * qq + 2 * i], sc[i], sh[i]);
          float f1 = fmaf(acc[j][4 * qq + 2 * i + 1], sc[i], sh[i]);
          if (g.relu) { f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f); }
          const __half2 h2 = __floats2half2_rn(f0, f1);
          v[mm] = *reinterpret_cast<const uint32_t*>(&h2);
        }
        stmatrix_x4_trans(lane_addr + (uint32_t)(((2 * wg + j) * 128 + q * 8) * kStemPitch), v);
      }
    named_sync(1, 256);
    // coalesced copy-out: 8 consecutive threads write one pixel's 128 bytes; pixels past the map's edge are clipped
#pragma unroll 4
    for (int i = ct; i < kStemTT * kStemTH * kStemTW * 8; i += 256) {
      const int pix = i >> 3, ch = i & 7;
      const int ot = tt * kStemTT + (pix >> 7), oh = th * kStemTH + ((pix >> 3) & 15), ow = tw * kStemTW + (pix & 7);
      if (ot >= g.OT || oh >= g.OH || ow >= g.OW) continue;
      const uint4 val = *reinterpret_cast<const uint4*>(ring + (size_t)pix * kStemPitch + ch * 16);
      *reinterpret_cast<uint4*>(y + ((((size_t)n * g.OT + ot) * g.OH + oh) * g.OW + ow) * g.out_ld + g.out_coff + ch * 8) = val;
    }
  }
}

// ---- host -------------------------------------------------------------------------------------
// The s2d stem: 24 input channels, 64 output channels, 4x4x4 taps, pad 1, stride 1, and the zero weights of the last t tap
// plane's channels >= 16 that the kernel does not multiply.
bool conv3d_stem_supported(const step_conv_params* p) {
  return p->dtype == STEP_F16 && p->Cin == 24 && p->Cout == 64 && p->KT == 4 && p->KH == 4 && p->KW == 4 && p->ST == 1 &&
         p->SH == 1 && p->SW == 1 && p->PT == 1 && p->PH == 1 && p->PW == 1 && p->OT == p->T && p->OH == p->H &&
         p->OW == p->W && !p->residual && p->n_splits == 0 && p->zero_cin_last_kt > 0 && p->zero_cin_last_kt <= 16;
}

int conv3d_stem_launch(const step_conv_params* p, step_stream_t stream) {
  STEP_CHECK_ARG(conv3d_stem_supported(p), "conv3d(stem): unsupported problem");
  STEP_CHECK_ARG((((uintptr_t)p->x | (uintptr_t)p->w | (uintptr_t)p->y) & 15) == 0 && p->in_ld % 8 == 0 && p->in_ld >= 24 &&
                 p->w_ld % 8 == 0 && p->w_ld >= 24 && p->out_ld % 8 == 0 && p->out_coff % 8 == 0, "conv3d(stem): alignment");
  StemGeom g;
  memset(&g, 0, sizeof(g));
  g.OT = p->OT; g.OH = p->OH; g.OW = p->OW;
  g.out_ld = p->out_ld; g.out_coff = p->out_coff; g.relu = p->relu;
  g.tiles_w = (p->OW + kStemTW - 1) / kStemTW; g.tiles_h = (p->OH + kStemTH - 1) / kStemTH;
  g.tiles_t = (p->OT + kStemTT - 1) / kStemTT;
  const long long ctas = (long long)p->N * g.tiles_t * g.tiles_h * g.tiles_w;
  STEP_CHECK_ARG(ctas < (1LL << 31), "conv3d(stem): grid too large");
  CUtensorMap mx, mw;
  // channels 24.. of the buffer lie outside the map: never read
  const cuuint32_t box[5] = {8, (cuuint32_t)kStemHpW, (cuuint32_t)kStemHpH, (cuuint32_t)kStemHpT, 1};
  if (int rc = encode_act5d(&mx, p->x, ActLayout(p->N, p->T, p->H, p->W, 24, p->in_ld), box, CU_TENSOR_MAP_SWIZZLE_NONE,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "conv3d(stem): patch"))
    return rc;
  // 64 output channels, 64 taps, 24 channels; boxes of one 8-channel group of one tap
  if (int rc = encode_weights3d(&mw, p->w, 64, 64, 24, p->w_ld, 8, 64, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "conv3d(stem): weights"))
    return rc;
  static std::atomic<unsigned long long> attr_seen{0};
  if (int rc = allow_dynamic_smem(conv_stem_kernel, attr_seen, kStemSmem, "conv_stem_kernel")) return rc;
  return launch_tc("conv_stem_kernel", conv_stem_kernel, dim3((unsigned)ctas), kStemThreads, kStemSmem, cu(stream), mx, mw, g,
                   p->scale, p->shift, (__half*)p->y);
}

}  // namespace step
