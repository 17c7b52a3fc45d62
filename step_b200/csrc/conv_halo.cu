// conv_halo.cu -- stride-1 k>1 convolution on thin inputs (Cin <= 64 channels: the 3x3x3 layers of the Mixed blocks'
// second branch; the space-to-depth I3D stem runs in conv_stem.cu) with the input neighbourhood staged ONCE in shared memory.
//
// The im2col path of conv_umma.cu fetches a fresh 128-row A tile from L2 for every filter tap; with 32 input channels a tap
// is a K=32 sliver and the kernel is bound by the bytes it pulls through TMA for each of them.  Here a CTA owns an output
// tile of TT x 16 x 8 pixels; BK/8 TMA box loads bring the (TT+KT-1) x (16+KH-1) x (8+KW-1) input patch (zero-filled outside
// the tensor == the TF-"SAME" halo, i3dpt.py:14-31) into shared memory, and every tap is TT wgmma sequences whose A
// descriptor simply starts at the tap's pixel offset inside the patch.
//
// Patch layout: the wgmma no-swizzle K-major layout, [BK/8 channel groups][pixel (t, h, w)][8 channels = 16 bytes].  A core
// matrix (8 rows x 16 bytes) is 8 consecutive w pixels of one channel group, so the operand of a tap starts at any pixel:
// LBO (next 8 channels) = one channel group's bytes, SBO (next 8-row group = next h row of the tile) = the patch row pitch.
// Only the weights (Cout x Cin per tap) stream through a TMA ring (128B / 64B / 32B swizzled like conv_umma.cu).
//
// Warp roles (384 threads): warp 0 producer (patch + weight ring), warpgroups 1 and 2 consume output rows h 0-7 / 8-15 of the
// tile for all TT planes (registers: TT x BN / 2 accumulators) and store the BN scale/shift + ReLU epilogue directly.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "umma_ptx.cuh"

namespace step {

constexpr int kHaloThreads = 384;
constexpr int kHaloTH = 16, kHaloTW = 8;   // 128 output pixels = two m64 warpgroups
constexpr int kHaloMaxStages = 16;
constexpr int kHaloSmemMax = 227 * 1024;
constexpr int kHaloBook = 4096;            // barriers (first 512 B), scale, shift

struct HaloGeom {
  int KT, KH, KW, PT, PH, PW, taps;
  int hp_t, hp_h, hp_w;          // patch extent in pixels
  int chunk_bytes;               // one 8-channel group of the patch, padded to 128 bytes
  int patch_bytes, b_bytes, n_stages;
  int Cout, relu, out_ld, out_coff;
  int tiles_w, tiles_h, tiles_t, OT, OH, OW;
};

template <int BK, int NCH, int TT>
__global__ void __launch_bounds__(kHaloThreads, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, HaloGeom g,
                 const float* __restrict__ scale, const float* __restrict__ shift, __half* __restrict__ y) {
  constexpr int BN = NCH * 64;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint64_t* full_bar = (uint64_t*)smem_raw;            // [kHaloMaxStages] weight stage landed
  uint64_t* empty_bar = full_bar + kHaloMaxStages;     // [kHaloMaxStages] weight stage consumed
  uint64_t* pfull_bar = empty_bar + kHaloMaxStages;    // patch landed
  float* s_scale = (float*)(smem_raw + 512);           // [BN <= 128]
  float* s_shift = s_scale + 128;
  uint8_t* ring = (uint8_t*)(((uintptr_t)smem_raw + kHaloBook + 1023) & ~(uintptr_t)1023);
  uint8_t* patch = ring + (size_t)g.n_stages * g.b_bytes;   // 1024-aligned: b_bytes is a multiple of 1024

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int b = blockIdx.x;
  const int tw = b % g.tiles_w; b /= g.tiles_w;
  const int th = b % g.tiles_h; b /= g.tiles_h;
  const int tt = b % g.tiles_t;
  const int n = b / g.tiles_t;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    for (int s = 0; s < g.n_stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_init(pfull_bar, 1);
    fence_barrier_init();
  }
  if (threadIdx.x < 128) {
    for (int i = threadIdx.x; i < BN; i += 128) {
      s_scale[i] = (scale && i < g.Cout) ? scale[i] : 1.0f;
      s_shift[i] = (shift && i < g.Cout) ? shift[i] : 0.0f;
    }
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== producer =====================
    if (elect_one()) {
      mbar_expect_tx(pfull_bar, (uint32_t)((BK / 8) * g.hp_t * g.hp_h * g.hp_w * 16));   // bytes TMA writes (without padding)
      for (int c = 0; c < BK / 8; ++c)
        tma_load_5d(&map_a, pfull_bar, patch + (size_t)c * g.chunk_bytes, c * 8, tw * kHaloTW - g.PW, th * kHaloTH - g.PH,
                    tt * TT - g.PT, n);
      for (int tap = 0; tap < g.taps; ++tap) {
        const int s = tap % g.n_stages, use = tap / g.n_stages;
        if (use > 0) mbar_wait(&empty_bar[s], (uint32_t)(use - 1) & 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)g.b_bytes);
        tma_load_3d(&map_b, &full_bar[s], ring + (size_t)s * g.b_bytes, 0, tap, 0);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers =====================
    const int wg = (warp >> 2) - 1;                      // output rows h = 8 wg .. 8 wg + 7 of the tile
    const int ct = threadIdx.x - 128;
    const uint64_t a_hi = ((uint64_t)((uint32_t)g.chunk_bytes >> 4) << 16) | ((uint64_t)((uint32_t)(g.hp_w * 16) >> 4) << 32);
    const uint64_t b_hi = desc_hi_kmajor<BK>();
    const uint64_t patch_lo = desc_lo(patch), ring_lo = desc_lo(ring);
    const uint32_t chunk16 = (uint32_t)g.chunk_bytes >> 4, plane16 = (uint32_t)(g.hp_h * g.hp_w), b16 = (uint32_t)g.b_bytes >> 4;
    float acc[TT * NCH * 32];                            // plane j: acc[j * NCH * 32 ...]; zeroed by the first tap
    mbar_wait(pfull_bar, 0);
    int kw = 0, kh = 0, kt = 0, s = 0, prev = -1;
    uint32_t par = 0;
    for (int tap = 0; tap < g.taps; ++tap) {
      mbar_wait(&full_bar[s], par);
      // one 16-byte pixel row of the patch == 1 in descriptor units
      const uint64_t a_lo = patch_lo + (uint64_t)((kt * g.hp_h + kh + 8 * wg) * g.hp_w + kw);
      const uint64_t b_lo = ring_lo + (uint64_t)s * b16;
      wg_fence();
#pragma unroll
      for (int j = 0; j < TT; ++j)
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
#pragma unroll
          for (int c = 0; c < NCH; ++c)
            wgmma_64x64(acc + (j * NCH + c) * 32, a_hi | (a_lo + (uint64_t)(j * plane16 + 2 * k * chunk16)),
                        b_hi | (b_lo + (uint64_t)(c * ((64 * BK * 2) >> 4)) + 2 * k), (tap | k) ? 1u : 0u);
      wg_commit();
      wg_wait<1>();
      if (prev >= 0 && ct % 128 == 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++kw == g.KW) { kw = 0; if (++kh == g.KH) { kh = 0; ++kt; } }
      if (++s == g.n_stages) { s = 0; par ^= 1u; }
    }
    wg_wait<0>();
    // epilogue: thread rows h = 8 wg + 2 (warp % 4) + i, w = lane / 4; columns 8 j + 2 (lane % 4) + {0, 1}
    const int ow = tw * kHaloTW + (lane >> 2);
#pragma unroll
    for (int j = 0; j < TT; ++j) {
      const int ot = tt * TT + j;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int oh = th * kHaloTH + 8 * wg + 2 * (warp & 3) + i;
        if (ot >= g.OT || oh >= g.OH || ow >= g.OW) continue;
        __half* dst = y + ((((size_t)n * g.OT + ot) * g.OH + oh) * g.OW + ow) * g.out_ld + g.out_coff;
#pragma unroll
        for (int q = 0; q < NCH * 8; ++q) {
          const int col = 8 * q + 2 * (lane & 3);
          if (col >= g.Cout) continue;
          float f0 = fmaf(acc[j * NCH * 32 + 4 * q + 2 * i], s_scale[col], s_shift[col]);
          float f1 = fmaf(acc[j * NCH * 32 + 4 * q + 2 * i + 1], s_scale[col + 1], s_shift[col + 1]);
          if (g.relu) { f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f); }
          *reinterpret_cast<__half2*>(dst + col) = __floats2half2_rn(f0, f1);
        }
      }
    }
  }
}

// ---- host -------------------------------------------------------------------------------------
// Does this problem fit the kernel?  (stride 1 is checked by the caller)
bool conv3d_halo_supported(const step_conv_params* p) {
  const int taps = p->KT * p->KH * p->KW;
  return p->dtype == STEP_F16 && taps > 1 && (p->Cin == 16 || p->Cin == 32 || p->Cin == 64) && p->in_ld % 8 == 0 &&
         p->Cout % 8 == 0 && p->Cout <= 256 && !p->residual && p->n_splits == 0 && p->KT <= 8 && p->KH <= 8 && p->KW <= 8 &&
         p->OT == p->T && p->OH == p->H && p->OW == p->W;
}

template <int BK, int NCH, int TT>
static int launch_halo_tt(const CUtensorMap& ma, const CUtensorMap& mb, const HaloGeom& g, size_t smem, unsigned grid,
                          const step_conv_params* p, const float* scale, const float* shift, __half* y, cudaStream_t s) {
  static std::atomic<unsigned long long> attr_seen{0};
  if (int rc = allow_dynamic_smem(conv_halo_kernel<BK, NCH, TT>, attr_seen, kHaloSmemMax, "conv_halo_kernel")) return rc;
  return launch_tc("conv_halo_kernel", conv_halo_kernel<BK, NCH, TT>, dim3(grid), kHaloThreads, smem, s, ma, mb, g, scale,
                   shift, y);
}

template <int BK>
static int launch_halo(const CUtensorMap& ma, const CUtensorMap& mb, const HaloGeom& g, int nch, int TT, size_t smem,
                       unsigned grid, const step_conv_params* p, cudaStream_t s) {
  const float* sc = p->scale;
  const float* sh = p->shift;
  __half* y = (__half*)p->y;
  if (nch == 1) {
    if (TT == 4) return launch_halo_tt<BK, 1, 4>(ma, mb, g, smem, grid, p, sc, sh, y, s);
    if (TT == 2) return launch_halo_tt<BK, 1, 2>(ma, mb, g, smem, grid, p, sc, sh, y, s);
    return launch_halo_tt<BK, 1, 1>(ma, mb, g, smem, grid, p, sc, sh, y, s);
  }
  if (TT == 2) return launch_halo_tt<BK, 2, 2>(ma, mb, g, smem, grid, p, sc, sh, y, s);
  return launch_halo_tt<BK, 2, 1>(ma, mb, g, smem, grid, p, sc, sh, y, s);
}

// one column tile of <= 128 output channels (weights and scale / shift offset by the tile's first channel)
static int halo_launch_cols(const step_conv_params* p, int c0, int cout, step_stream_t stream) {
  const int BK = p->Cin, row = BK * 2;
  HaloGeom g;
  memset(&g, 0, sizeof(g));
  g.KT = p->KT; g.KH = p->KH; g.KW = p->KW; g.PT = p->PT; g.PH = p->PH; g.PW = p->PW; g.taps = p->KT * p->KH * p->KW;
  g.Cout = cout; g.relu = p->relu; g.OT = p->OT; g.OH = p->OH; g.OW = p->OW;
  g.out_ld = p->out_ld; g.out_coff = p->out_coff + c0;
  const int nch = cout <= 64 ? 1 : 2;
  const int BN = nch * 64;
  // Output planes per CTA (accumulator sets in registers, TT * BN <= 256).  Every tap's weight tile is fetched once per CTA,
  // so more planes mean less weight traffic per pixel; the patch for TT planes plus >= 2 weight stages must fit 227 KB.
  int best_tt = 1;
  for (int tt = 256 / BN > 4 ? 4 : 256 / BN; tt > 1; tt >>= 1) {
    const long patch = (long)(tt + g.KT - 1) * (kHaloTH + g.KH - 1) * (kHaloTW + g.KW - 1) * row;
    if (kHaloBook + 1024 + patch + 2L * BN * row > kHaloSmemMax) continue;
    // prefer the larger tile unless more than a quarter of the computed planes would fall past the end
    const int groups = (p->OT + tt - 1) / tt;
    if ((groups * tt - p->OT) * 4 > groups * tt) continue;
    best_tt = tt;
    break;
  }
  const int TT = best_tt;
  g.hp_t = TT + g.KT - 1; g.hp_h = kHaloTH + g.KH - 1; g.hp_w = kHaloTW + g.KW - 1;
  g.chunk_bytes = (g.hp_t * g.hp_h * g.hp_w * 16 + 127) / 128 * 128;   // TMA destinations are 128-byte aligned
  g.patch_bytes = (BK / 8) * g.chunk_bytes;
  g.b_bytes = BN * row;
  long n_st = ((long)kHaloSmemMax - kHaloBook - 1024 - g.patch_bytes) / g.b_bytes;
  STEP_CHECK_ARG(n_st >= 2, "conv3d(halo): patch of %d bytes leaves no room for the weight ring", g.patch_bytes);
  if (n_st > kHaloMaxStages) n_st = kHaloMaxStages;
  if (n_st > g.taps) n_st = g.taps;
  g.n_stages = (int)n_st;
  g.tiles_w = (p->OW + kHaloTW - 1) / kHaloTW; g.tiles_h = (p->OH + kHaloTH - 1) / kHaloTH; g.tiles_t = (p->OT + TT - 1) / TT;
  const long long ctas = (long long)p->N * g.tiles_t * g.tiles_h * g.tiles_w;
  STEP_CHECK_ARG(ctas < (1LL << 31), "conv3d(halo): grid too large");
  const size_t smem = kHaloBook + 1024 + (size_t)g.n_stages * g.b_bytes + (size_t)g.patch_bytes;
  STEP_CHECK_ARG(smem <= (size_t)kHaloSmemMax, "conv3d(halo): %zu bytes of shared memory", smem);
  CUtensorMap ma, mb;
  const cuuint32_t box[5] = {8, (cuuint32_t)g.hp_w, (cuuint32_t)g.hp_h, (cuuint32_t)g.hp_t, 1};
  if (int rc = encode_act5d(&ma, p->x, ActLayout(p->N, p->T, p->H, p->W, p->Cin, p->in_ld), box, CU_TENSOR_MAP_SWIZZLE_NONE,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "conv3d(halo): patch"))
    return rc;
  const __half* w = (const __half*)p->w + (size_t)c0 * g.taps * p->w_ld;
  if (int rc = encode_weights3d(&mb, w, cout, g.taps, p->Cin, p->w_ld, BK, BN, swizzle_for(BK),
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "conv3d(halo): weights"))
    return rc;
  step_conv_params q = *p;
  q.scale = p->scale ? p->scale + c0 : nullptr;
  q.shift = p->shift ? p->shift + c0 : nullptr;
  if (BK == 64) return launch_halo<64>(ma, mb, g, nch, TT, smem, (unsigned)ctas, &q, cu(stream));
  if (BK == 32) return launch_halo<32>(ma, mb, g, nch, TT, smem, (unsigned)ctas, &q, cu(stream));
  return launch_halo<16>(ma, mb, g, nch, TT, smem, (unsigned)ctas, &q, cu(stream));
}

int conv3d_halo_launch(const step_conv_params* p, step_stream_t stream) {
  STEP_CHECK_ARG(conv3d_halo_supported(p) && p->ST == 1 && p->SH == 1 && p->SW == 1, "conv3d(halo): unsupported problem");
  STEP_CHECK_ARG((((uintptr_t)p->x | (uintptr_t)p->w | (uintptr_t)p->y) & 15) == 0 && p->w_ld % 8 == 0 && p->w_ld >= p->Cin &&
                 p->out_ld % 8 == 0 && p->out_coff % 8 == 0, "conv3d(halo): alignment");
  // more than 128 output channels: launches of 128-column tiles (registers hold at most 64 accumulators per thread)
  for (int c0 = 0; c0 < p->Cout; c0 += 128) {
    const int cout = p->Cout - c0 < 128 ? p->Cout - c0 : 128;
    if (int rc = halo_launch_cols(p, c0, cout, stream)) return rc;
  }
  return 0;
}

}  // namespace step
