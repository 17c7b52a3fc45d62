// conv_umma.cu -- channels-last 3-D / 2-D convolution as an implicit GEMM on the Hopper tensor cores (sm_90a):
// TMA-staged operand tiles, wgmma with the fp32 accumulator in registers, fused BatchNorm-scale/shift (+bias) + residual
// + ReLU epilogue that writes a channel slice of a wider buffer (the Inception concat, models/i3dpt.py:157-163, never
// materialises) or scatters column ranges to up to three destinations (horizontally fused 1x1x1 layers).
//
// Replaces, for the fp16 path, every Conv3d/BatchNorm3d/ReLU triple of models/i3dpt.py:103-111 and
// the Conv2d/ReLU/residual chains of models/two_branch.py:60-111,236,258.
//
// GEMM view:  D[M = output pixels, N = Cout] = A[M, K = taps x Cin] * B[K, N]
//   A (activations, [N,T,H,W,Cin] fp16, K-major rows = pixels): one TMA load per (filter tap,
//     channel block) into a 128-row swizzled tile.  Three addressing modes:
//       LINEAR  1x1x1 filters: the tensor is a plain [M, Cin] matrix (2-D map), dense M tiles.
//       BOX     k>1: the M tile is a (bw x bh x bt) box of output pixels; the tap shifts the box and
//               TMA zero-fills out-of-bounds pixels == the TF-"SAME" zero halo (i3dpt.py:14-31).
//       IM2COL  k>1: TMA im2col mode walks 128 consecutive output pixels (w->h->t->n) inside the
//               padded bounding box; dense M tiles on any map size.
//   B (weights, [Cout, taps, Cin] fp16, K-major rows = output channels): 3-D map, box (BK,1,BN).
//   D: fp32 in registers; consumer warpgroup w owns rows [64 w, 64 w + 64) x BN columns (BN / 2 registers), and issues one
//      m64nBNk16 wgmma per 16-element K step.  BN is sized to Cout (up to 256, see pick_tile).
// Persistent: CTA b runs tiles b, b + grid, b + 2 grid, ... with no CTA waiting on another (tiles with long K loops get one
// CTA each, see build_plan).
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected thread of warp 0) and, in warps 1-3, the copy-out of
// the fp16 output staging tile to global plus the next tile's epilogue constants; warpgroups 1, 2 = wgmma consumers and
// the register half of the epilogue; for BN > 128 warpgroup 0 hands registers to the consumers (setmaxnreg).  Pipeline:
// n_stages smem stages with full / empty mbarriers, carried across tiles, so the producer loads the next tile while the
// epilogue of this one runs.  The staging tile is a buffer of its own, handed between consumers and copy warps by one
// full / empty mbarrier pair.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "umma_ptx.cuh"

namespace step {

constexpr int kBM = 128;       // two m64 warpgroups
constexpr int kMaxBN = 256;    // 128 fp32 accumulator registers per consumer thread
constexpr int kStages = 8;     // barrier slots
constexpr int kThreads = 384;
constexpr int kConsumers = 256;
constexpr int kCopyThreads = 96;  // warps 1-3
constexpr int kPersistMaxKBlocks = 100;  // longer K loops run one tile per CTA (build_plan)
// stage barriers, staging-tile barriers, scale and shift of two consecutive tiles
constexpr int kBookBytes = 2 * kStages * 8 + 2 * 8 + 2 * 2 * kMaxBN * 4;
// registers per thread after the hand-over of wide tiles: 128 x 40 + 256 x 232 = 384 x 168, the launch allocation
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

// (BK, BN) instantiations of conv_umma_kernel: exactly the tiles pick_bk / pick_tile choose for the C4 layer table
// (DESIGN.md section 3.1), plus (16, 64) for Cin <= 16, which the C4 step sends to the patch kernel (conv_halo.cu).  The
// 64-column tile of each BK serves every other Cout, with padded columns.
#define STEP_CONV_TILES(X)                                                                                         \
  X(64, 32) X(64, 64) X(64, 128) X(64, 144) X(64, 152) X(64, 176) X(64, 192) X(64, 208) X(64, 224) X(64, 256)      \
  X(32, 64) X(32, 128) X(32, 144) X(32, 152) X(32, 160) X(32, 208) X(32, 224)                                      \
  X(16, 64)

// byte pitch of a row of the fp16 output staging tile: BN columns plus 16 bytes, rounded up to an odd multiple of 16
// so that the 8 rows one store instruction touches spread over the banks
__host__ __device__ constexpr int staging_pitch(int BN) { return ((BN / 8 + 1) | 1) * 16; }

struct ConvGeom {
  int mode;
  int taps, KT, KH, KW, PT, PH, PW;
  int kblocks_per_tap;          // ceil(Cin / BK); the channel tail of a tap's last block is TMA zero fill in A and B
  int BN, n_tiles;              // N tile (a STEP_CONV_TILES width) and count
  int n_stages;                 // smem pipeline depth
  int n_splits, split[2], ld_extra[2], coff_extra[2];  // fused 1x1x1 layers: extra destinations by column range
  __half* y_extra[2];
  int Cout, out_ld, out_coff, res_ld, res_coff, relu;
  int OT, OH, OW, Nimg;
  long long M;                  // Nimg*OT*OH*OW
  int tiles;                    // M tiles x n_tiles
  int bw, bh, bt, tiles_w, tiles_h, tiles_t;  // BOX mode
  int a_bytes;                  // bytes TMA writes for A per stage
};

// output pixel of row `row` of M tile `m_tile`, or -1 (past the end / box overhang)
__device__ __forceinline__ long long tile_row_pixel(const ConvGeom& g, int m_tile, int row) {
  if (g.mode == STEP_A_BOX) {
    int r = m_tile;
    const int bw0 = (r % g.tiles_w) * g.bw; r /= g.tiles_w;
    const int bh0 = (r % g.tiles_h) * g.bh; r /= g.tiles_h;
    const int bt0 = (r % g.tiles_t) * g.bt; const int bn = r / g.tiles_t;
    const int dw = row % g.bw, rr = row / g.bw;
    const int dh = rr % g.bh, dt = rr / g.bh;
    const int ow = bw0 + dw, oh = bh0 + dh, ot = bt0 + dt;
    if (dt < g.bt && ow < g.OW && oh < g.OH && ot < g.OT) return (((long long)bn * g.OT + ot) * g.OH + oh) * g.OW + ow;
    return -1;
  }
  const long long m = (long long)m_tile * kBM + row;
  return m < g.M ? m : -1;
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return done != 0;
}

// ---- the kernel -----------------------------------------------------------------------------
template <int BK, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, ConvGeom g,
                 const float* __restrict__ scale, const float* __restrict__ shift, const __half* __restrict__ residual,
                 __half* __restrict__ y) {
  static_assert(BN % 8 == 0 && BN <= kMaxBN, "wgmma N is a multiple of 8, at most 256");
  // more than 64 accumulators per consumer thread do not fit the even share of the register file (168 per thread)
  constexpr bool kRealloc = BN > 128;
  // rows of more than 256 bytes leave the staging tile as bulk copies; per-copy overhead makes narrower rows faster as
  // 16-byte stores
  constexpr bool kBulkOut = BN > 128;
  constexpr int kABytes = kBM * BK * 2;
  constexpr int kBBytes = BN * BK * 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stage barriers | staging barriers | scale, shift x 2] (kBookBytes) then the 1024-aligned stage area
  // [A stages][B stages], then the fp16 output staging tile (kBM rows of staging_pitch(BN) bytes).
  uint64_t* full_bar = (uint64_t*)smem_raw;
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* out_full = empty_bar + kStages;     // phase 1 of the CTA's i-th tile has written the staging tile
  uint64_t* out_empty = out_full + 1;           // the copy warps have read the i-th tile out of it
  // scale and shift of the CTA's i-th tile live in buffer i & 1: the copy warps stage tile i + 1 while tile i's
  // epilogue may still read buffer i & 1
  float* s_consts = (float*)(out_empty + 1);    // [2][scale BN | shift BN] with kMaxBN pitch
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + kBookBytes + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + g.n_stages * kABytes;
  uint8_t* stg = smem + g.n_stages * (kABytes + kBBytes);
  constexpr int pitch = staging_pitch(BN);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = g.taps * g.kblocks_per_tap;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    mbar_init(out_full, kConsumers / 32);
    mbar_init(out_empty, kCopyThreads / 32);
    fence_barrier_init();
  }
  // the per-channel epilogue constants of N tile n_tile into buffer `buf`, by `nthr` threads starting at `t`
  auto stage_consts = [&](int n_tile, int buf, int t, int nthr) {
    float* s_scale = s_consts + buf * 2 * kMaxBN;
    float* s_shift = s_scale + kMaxBN;
    for (int i = t; i < BN; i += nthr) {
      const int c = n_tile * BN + i;
      s_scale[i] = (scale && c < g.Cout) ? scale[c] : 1.0f;
      s_shift[i] = (shift && c < g.Cout) ? shift[c] : 0.0f;
    }
  };
  if (threadIdx.x < 128) stage_consts(blockIdx.x % g.n_tiles, 0, threadIdx.x, 128);
  __syncthreads();

  if (warp < 4) {
    if constexpr (kRealloc) setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // ===================== TMA producer =====================
      if (elect_one()) {
        const uint32_t tx_bytes = (uint32_t)(g.a_bytes + kBBytes);
        int stage = 0; uint32_t phase = 0;       // carried from each tile's last k-block into the next tile's first
        for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
          const int m_tile = tile / g.n_tiles, n0 = (tile - m_tile * g.n_tiles) * BN;
          long long m0 = (long long)m_tile * kBM;
          int bn = 0, bt0 = 0, bh0 = 0, bw0 = 0;  // BOX origin
          if (g.mode == STEP_A_BOX) {
            int r = m_tile;
            bw0 = (r % g.tiles_w) * g.bw; r /= g.tiles_w;
            bh0 = (r % g.tiles_h) * g.bh; r /= g.tiles_h;
            bt0 = (r % g.tiles_t) * g.bt; bn = r / g.tiles_t;
          }
          // IM2COL start coordinates: output pixel m0 -> (w,h,t,n) + lower corner (= -pad)
          int iw = 0, ih = 0, it = 0, in_ = 0;
          if (g.mode == STEP_A_IM2COL) {
            long long r = m0;
            iw = (int)(r % g.OW); r /= g.OW;
            ih = (int)(r % g.OH); r /= g.OH;
            it = (int)(r % g.OT); in_ = (int)(r / g.OT);
            iw -= g.PW; ih -= g.PH; it -= g.PT;
          }
          int kw = 0, kh = 0, kt = 0;                // filter tap, advanced incrementally (no divisions in the loop)
          for (int tap = 0; tap < g.taps; ++tap) {
            for (int kc = 0; kc < g.kblocks_per_tap; ++kc) {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              mbar_expect_tx(&full_bar[stage], tx_bytes);
              const int c0 = kc * BK;
              uint8_t* a_dst = sA + stage * kABytes;
              if (g.mode == STEP_A_LINEAR) {
                tma_load_2d(&map_a, &full_bar[stage], a_dst, c0, (int)m0);
              } else if (g.mode == STEP_A_BOX) {
                tma_load_5d(&map_a, &full_bar[stage], a_dst, c0, bw0 + kw - g.PW, bh0 + kh - g.PH, bt0 + kt - g.PT, bn);
              } else {
                tma_load_im2col_5d(&map_a, &full_bar[stage], a_dst, c0, iw, ih, it, in_, (uint16_t)kw, (uint16_t)kh,
                                   (uint16_t)kt);
              }
              tma_load_3d(&map_b, &full_bar[stage], sB + stage * kBBytes, c0, tap, n0);
              if (++stage == g.n_stages) { stage = 0; phase ^= 1; }
            }
            if (++kw == g.KW) { kw = 0; if (++kh == g.KH) { kh = 0; ++kt; } }
          }
        }
      }
    } else {
      // ===================== copy-out (warps 1-3) =====================
      const int ct = threadIdx.x - 32;           // 0..95
      int i_tile = 0;
      for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x, ++i_tile) {
        const int m_tile = tile / g.n_tiles, n0 = (tile - m_tile * g.n_tiles) * BN;
        // tile i - 1's phase 1, the last reader of buffer (i + 1) & 1, completed out_full before this thread's last wait
        if (tile + (int)gridDim.x < g.tiles) stage_consts((tile + gridDim.x) % g.n_tiles, (i_tile + 1) & 1, ct, kCopyThreads);
        // the copy warps sleep through the K loop instead of taking issue slots from the consumers
        while (!mbar_try_wait(out_full, i_tile & 1)) __nanosleep(128);
        if constexpr (!kBulkOut) {
          // Phase 2, narrow rows: coalesced copy-out, consecutive threads write consecutive 16-byte chunks of an output
          // row, kUnroll shared-memory loads in flight per thread
          constexpr int cpr = BN / 8;  // 16-byte chunks per row
          constexpr int kUnroll = 4;
          for (int i0 = ct; i0 < kBM * cpr; i0 += kUnroll * kCopyThreads) {
            uint4 val[kUnroll];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
              const int i = i0 + u * kCopyThreads, rr = i / cpr, ch = i - rr * cpr;
              if (i < kBM * cpr) val[u] = *reinterpret_cast<const uint4*>(stg + (size_t)rr * pitch + ch * 16);
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
              const int i = i0 + u * kCopyThreads, rr = i / cpr, ch = i - rr * cpr;
              const int col = n0 + ch * 8;
              if (i >= kBM * cpr || col >= g.Cout) continue;
              const long long rp = tile_row_pixel(g, m_tile, rr);
              if (rp < 0) continue;
              __half* dst = y + (size_t)rp * g.out_ld + g.out_coff + col;
              if (g.n_splits > 0 && col >= g.split[0]) {
                const int d = (g.n_splits > 1 && col >= g.split[1]) ? 1 : 0;
                dst = g.y_extra[d] + (size_t)rp * g.ld_extra[d] + g.coff_extra[d] + (col - g.split[d]);
              }
              *reinterpret_cast<uint4*>(dst) = val[u];
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(out_empty);
          continue;
        }
        // Phase 2, wide rows: one bulk copy (TMA engine) per output row and destination: the row's columns
        // [n0, min(n0 + BN, Cout)) cut at the split columns (multiples of 16, so every piece stays 16-byte aligned); box
        // overhang rows are skipped.
        const int end = min(n0 + BN, g.Cout);
        for (int rr = ct; rr < kBM; rr += kCopyThreads) {
          const long long rp = tile_row_pixel(g, m_tile, rr);
          if (rp < 0) continue;
          for (int col = n0; col < end;) {
            __half* dst = y + (size_t)rp * g.out_ld + g.out_coff + col;
            int next = end;
            if (g.n_splits > 0) {
              if (col >= g.split[0]) {
                const int d = (g.n_splits > 1 && col >= g.split[1]) ? 1 : 0;
                dst = g.y_extra[d] + (size_t)rp * g.ld_extra[d] + g.coff_extra[d] + (col - g.split[d]);
                if (d == 0 && g.n_splits > 1) next = min(end, g.split[1]);
              } else {
                next = min(end, g.split[0]);
              }
            }
            bulk_store(dst, stg + (size_t)rr * pitch + (col - n0) * 2, (uint32_t)(next - col) * 2);
            col = next;
          }
        }
        bulk_commit();
        bulk_wait_read<0>();                     // the staging tile has been read
        // staging reads and the next tile's constants are ordered before the arrival
        __syncwarp();
        if (lane == 0) mbar_arrive(out_empty);
      }
    }
  } else {
    // ===================== consumers (warpgroups 1, 2) =====================
    if constexpr (kRealloc) setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;              // 64-row half of the tile
    const int ct = threadIdx.x - 128;            // 0..255
    const uint64_t hi = desc_hi_kmajor<BK>();
    const uint64_t a_lo0 = desc_lo(sA + wg * 64 * BK * 2), b_lo0 = desc_lo(sB);
    const int wrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;           // carried across tiles, as in the producer
    int i_tile = 0;
    for (int tile = blockIdx.x; tile < g.tiles; tile += gridDim.x, ++i_tile) {
      const int m_tile = tile / g.n_tiles, n0 = (tile - m_tile * g.n_tiles) * BN;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t a_lo = a_lo0 + (uint64_t)(stage * (kABytes >> 4)), b_lo = b_lo0 + (uint64_t)(stage * (kBBytes >> 4));
        wg_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)        // 16 elements (32 bytes) along K inside the swizzle atom per step
          wgmma_f16<BN>(acc, hi | (a_lo + 2 * k), hi | (b_lo + 2 * k), 1u);
        wg_commit();
        wg_wait<1>();                            // the previous k-block's MMAs have retired: free its stage
        if (prev >= 0 && ct % 128 == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == g.n_stages) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      if (ct % 128 == 0) mbar_arrive(&empty_bar[prev]);  // the last stage too: the producer is filling the next tile
      // the copy warps have read the previous tile out of the staging tile
      mbar_wait(out_empty, (i_tile & 1) ^ 1);
      // Phase 1: registers -> scale/shift (+residual) (+relu) -> fp16 -> staging row.
      const float* s_scale = s_consts + (i_tile & 1) * 2 * kMaxBN;
      const float* s_shift = s_scale + kMaxBN;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = wrow + 8 * i;
        const long long pix = residual ? tile_row_pixel(g, m_tile, row) : -1;
        const __half* rrow = pix >= 0 ? residual + (size_t)pix * g.res_ld + g.res_coff + n0 : nullptr;
        uint8_t* srow = stg + (size_t)row * pitch;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          float f0 = fmaf(acc[4 * j + 2 * i], s_scale[col], s_shift[col]);
          float f1 = fmaf(acc[4 * j + 2 * i + 1], s_scale[col + 1], s_shift[col + 1]);
          if (rrow && n0 + col < g.Cout) {
            const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(rrow + col));
            f0 += rf.x; f1 += rf.y;
          }
          if (g.relu) { f0 = fmaxf(f0, 0.0f); f1 = fmaxf(f1, 0.0f); }
          *reinterpret_cast<__half2*>(srow + col * 2) = __floats2half2_rn(f0, f1);
        }
      }
      // hand the staging tile to the copy warps (Phase 2: bulk copies, which read it through the async proxy) and go on
      // with the next tile's K loop
      if constexpr (kBulkOut) fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(out_full);
    }
  }
}

// debug: load one A tile (tap kt,kh,kw, channel block c0) for m_tile and dump the raw stage bytes
template <int BK>
__global__ void __launch_bounds__(32) tma_dump_kernel(const __grid_constant__ CUtensorMap map_a, ConvGeom g, int m_tile,
                                                      int kt, int kh, int kw, int c0, uint8_t* __restrict__ out) {
  constexpr int kABytes = kBM * BK * 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t bar;
  for (int i = threadIdx.x; i < kABytes / 4; i += 32) ((uint32_t*)smem)[i] = 0xFFFFFFFFu;  // "never written"
  if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_barrier_init(); }
  fence_proxy_async();
  __syncwarp();
  if (threadIdx.x == 0) {
    long long m0 = (long long)m_tile * kBM;
    mbar_expect_tx(&bar, (uint32_t)g.a_bytes);
    if (g.mode == STEP_A_LINEAR) {
      tma_load_2d(&map_a, &bar, smem, c0, (int)m0);
    } else if (g.mode == STEP_A_BOX) {
      int r = m_tile;
      int bw0 = (r % g.tiles_w) * g.bw; r /= g.tiles_w;
      int bh0 = (r % g.tiles_h) * g.bh; r /= g.tiles_h;
      int bt0 = (r % g.tiles_t) * g.bt; int bn = r / g.tiles_t;
      tma_load_5d(&map_a, &bar, smem, c0, bw0 + kw - g.PW, bh0 + kh - g.PH, bt0 + kt - g.PT, bn);
    } else {
      long long r = m0;
      int iw = (int)(r % g.OW); r /= g.OW;
      int ih = (int)(r % g.OH); r /= g.OH;
      int it = (int)(r % g.OT); int in_ = (int)(r / g.OT);
      tma_load_im2col_5d(&map_a, &bar, smem, c0, iw - g.PW, ih - g.PH, it - g.PT, in_, (uint16_t)kw, (uint16_t)kh, (uint16_t)kt);
    }
  }
  mbar_wait(&bar, 0);
  __syncwarp();
  for (int i = threadIdx.x; i < kABytes / 4; i += 32) ((uint32_t*)out)[i] = ((uint32_t*)smem)[i];
}

// ---- host side --------------------------------------------------------------------------------
// Channel block width.  A tap's last block is zero-filled past Cin and its zero 16-channel steps are multiplied, not skipped
// (a data-dependent guard around the wgmma issue makes ptxas serialise the whole sequence), so the width is the one with
// the least padded K, the wider one on a tie: Cin = 96, 144, 160, 480, 528 -> blocks of 32 (no or less padding), 112 or
// 1088 -> 64.  Blocks of 16 only serve Cin <= 16.  The zero steps add exact zeros, so the choice does not change the result.
static int pick_bk(int Cin) {
  if (Cin <= 16) return 16;
  const int k64 = (Cin + 63) / 64 * 64, k32 = (Cin + 31) / 32 * 32;
  return k32 < k64 ? 32 : 64;
}

struct ConvTile {
  int BK, BN;
  void (*kernel)(CUtensorMap, CUtensorMap, ConvGeom, const float*, const float*, const __half*, __half*);
};
static const ConvTile kTiles[] = {
#define STEP_TILE_ENTRY(bk, bn) {bk, bn, conv_umma_kernel<bk, bn>},
    STEP_CONV_TILES(STEP_TILE_ENTRY)
#undef STEP_TILE_ENTRY
};
constexpr int kNumTiles = (int)(sizeof(kTiles) / sizeof(kTiles[0]));

// N tile for Cout among the instantiated widths of this BK: the fewest padded columns, then the fewest tiles
// (every N tile re-reads the whole A operand through L2).  E.g. 320 -> 2 x 160, 384 -> 2 x 192, 1024 -> 4 x 256.
static int pick_tile(int BK, int Cout) {
  int best = -1; long best_pad = 0, best_n = 0;
  for (int i = 0; i < kNumTiles; ++i) {
    if (kTiles[i].BK != BK) continue;
    const long n = (Cout + kTiles[i].BN - 1) / kTiles[i].BN, pad = n * kTiles[i].BN - Cout;
    if (best < 0 || pad < best_pad || (pad == best_pad && n < best_n)) { best = i; best_pad = pad; best_n = n; }
  }
  return best;
}

static void pick_box(int OW, int OH, int OT, int* bw, int* bh, int* bt) {
  double best = -1;
  for (int w = 1; w <= OW && w <= kBM; ++w)
    for (int h = 1; h <= OH && w * h <= kBM; ++h) {
      int t = kBM / (w * h);
      if (t > OT) t = OT;
      if (t < 1) continue;
      double eff = ((double)OW / (((OW + w - 1) / w) * w)) * ((double)OH / (((OH + h - 1) / h) * h)) *
                   ((double)OT / (((OT + t - 1) / t) * t)) * ((double)(w * h * t) / kBM);
      if (eff > best + 1e-9) { best = eff; *bw = w; *bh = h; *bt = t; }
    }
}

// Do two CTAs of tile `t` with `smem` bytes of dynamic shared memory fit one SM (registers included: the wide tiles that
// re-balance registers with setmaxnreg never do)?  The answer depends only on the instantiation (the caller derives `smem`
// from BK and BN), so it is asked once per instantiation.
static std::atomic<int> g_two_ctas[kNumTiles];                // 0 = not asked yet, 1 = no, 2 = yes
static std::atomic<unsigned long long> g_attr_seen[kNumTiles];

static int two_ctas_fit(int t, size_t smem, bool* two) {
  int v = g_two_ctas[t].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaError_t e = cudaFuncSetAttribute(kTiles[t].kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    int n = 0;
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kTiles[t].kernel, kThreads, smem);
    if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "conv3d(f16): occupancy query: %s", cudaGetErrorString(e)); }
    v = n >= 2 ? 2 : 1;
    g_two_ctas[t].store(v, std::memory_order_relaxed);
  }
  *two = v == 2;
  return 0;
}

// Streaming multiprocessors of the current device, asked once per device.
static std::atomic<int> g_sm_count[64];

static int sm_count(int* n) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "conv3d(f16): cudaGetDevice: %s", cudaGetErrorString(e)); }
  int v = g_sm_count[dev & 63].load(std::memory_order_relaxed);
  if (v == 0) {
    e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "conv3d(f16): SM count: %s", cudaGetErrorString(e)); }
    g_sm_count[dev & 63].store(v, std::memory_order_relaxed);
  }
  *n = v;
  return 0;
}

struct ConvPlan {
  CUtensorMap map_a, map_b;
  ConvGeom g;
  int BK;
  int tile;                     // index into kTiles
  size_t smem_bytes;
  dim3 grid;
};

static int build_plan(const step_conv_params* p, ConvPlan* pl) {
  STEP_CHECK_ARG(p->ST == 1 && p->SH == 1 && p->SW == 1, "conv3d(f16): stride must be 1 (use the s2d stem)");
  STEP_CHECK_ARG(p->Cin % 8 == 0 && p->in_ld % 8 == 0 && p->w_ld % 8 == 0 && p->w_ld >= p->Cin,
                 "conv3d(f16): Cin=%d in_ld=%d w_ld=%d must be multiples of 8", p->Cin, p->in_ld, p->w_ld);
  STEP_CHECK_ARG(p->Cout % 8 == 0 && p->out_ld % 8 == 0 && p->out_coff % 8 == 0, "conv3d(f16): Cout/out_ld/out_coff %% 8");
  STEP_CHECK_ARG(!p->residual || (p->res_ld % 8 == 0 && p->res_coff % 8 == 0), "conv3d(f16): res_ld/res_coff %% 8");
  STEP_CHECK_ARG((((uintptr_t)p->x | (uintptr_t)p->w | (uintptr_t)p->y | (uintptr_t)p->residual) & 15) == 0,
                 "conv3d(f16): pointers must be 16-byte aligned");
  ConvGeom& g = pl->g;
  memset(&g, 0, sizeof(g));
  const int taps = p->KT * p->KH * p->KW;
  const bool is_1x1 = taps == 1 && p->PT == 0 && p->PH == 0 && p->PW == 0 && p->OT == p->T && p->OH == p->H && p->OW == p->W;
  int mode = p->a_mode;
  if (mode == STEP_A_AUTO) mode = is_1x1 ? STEP_A_LINEAR : STEP_A_BOX;
  STEP_CHECK_ARG(mode == STEP_A_LINEAR || mode == STEP_A_BOX || mode == STEP_A_IM2COL, "conv3d(f16): bad a_mode %d", p->a_mode);
  STEP_CHECK_ARG(mode != STEP_A_LINEAR || is_1x1, "conv3d(f16): LINEAR mode needs a 1x1x1 unpadded filter");
  g.mode = mode;
  g.taps = taps; g.KT = p->KT; g.KH = p->KH; g.KW = p->KW; g.PT = p->PT; g.PH = p->PH; g.PW = p->PW;
  pl->BK = pick_bk(p->Cin);
  const int BK = pl->BK;
  g.kblocks_per_tap = (p->Cin + BK - 1) / BK;
  pl->tile = pick_tile(BK, p->Cout);
  g.BN = kTiles[pl->tile].BN;
  g.n_tiles = (p->Cout + g.BN - 1) / g.BN;
  g.Cout = p->Cout; g.out_ld = p->out_ld; g.out_coff = p->out_coff; g.res_ld = p->res_ld; g.res_coff = p->res_coff;
  g.relu = p->relu;
  g.n_splits = p->n_splits;
  if (p->n_splits) {
    STEP_CHECK_ARG(p->n_splits >= 1 && p->n_splits <= 2 && !p->residual, "conv3d(f16): fused outputs need no residual, 1-2 splits");
    int prev = 0;
    for (int i = 0; i < p->n_splits; ++i) {
      STEP_CHECK_ARG(p->split[i] % 16 == 0 && p->split[i] > prev && p->split[i] < p->Cout && p->y_extra[i] &&
                     p->ld_extra[i] % 8 == 0 && p->coff_extra[i] % 8 == 0 && ((uintptr_t)p->y_extra[i] & 15) == 0,
                     "conv3d(f16): bad split %d", i);
      prev = p->split[i];
      g.split[i] = p->split[i]; g.y_extra[i] = (__half*)p->y_extra[i]; g.ld_extra[i] = p->ld_extra[i]; g.coff_extra[i] = p->coff_extra[i];
    }
    STEP_CHECK_ARG(p->out_ld >= p->out_coff + p->split[0], "conv3d(f16): first destination too narrow");
  }
  g.OT = p->OT; g.OH = p->OH; g.OW = p->OW; g.Nimg = p->N;
  g.M = (long long)p->N * p->OT * p->OH * p->OW;
  long long m_tiles;
  int rc;
  if (mode == STEP_A_LINEAR) {
    STEP_CHECK_ARG(g.M < (1LL << 31), "conv3d(f16): M too large");
    rc = encode_rows2d(&pl->map_a, p->x, g.M, p->Cin, p->in_ld, BK, kBM, swizzle_for(BK), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       "conv3d(f16): A (linear)");
    m_tiles = (g.M + kBM - 1) / kBM;
    g.a_bytes = kBM * BK * 2;
  } else {
    const ActLayout act(p->N, p->T, p->H, p->W, p->Cin, p->in_ld);
    if (mode == STEP_A_BOX) {
      pick_box(p->OW, p->OH, p->OT, &g.bw, &g.bh, &g.bt);
      g.tiles_w = (p->OW + g.bw - 1) / g.bw; g.tiles_h = (p->OH + g.bh - 1) / g.bh; g.tiles_t = (p->OT + g.bt - 1) / g.bt;
      const cuuint32_t box[5] = {(cuuint32_t)BK, (cuuint32_t)g.bw, (cuuint32_t)g.bh, (cuuint32_t)g.bt, 1};
      rc = encode_act5d(&pl->map_a, p->x, act, box, swizzle_for(BK), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "conv3d(f16): A (box)");
      m_tiles = (long long)p->N * g.tiles_t * g.tiles_h * g.tiles_w;
      g.a_bytes = g.bw * g.bh * g.bt * BK * 2;
    } else {
      // TMA im2col: bounding box lower corner = -pad_low, upper corner = pad_high - (k-1)  (fprop, dilation 1);
      // rank-5 corners must lie in [-16, 15]
      const int ph_t = p->OT - p->T + p->KT - 1 - p->PT, ph_h = p->OH - p->H + p->KH - 1 - p->PH,
                ph_w = p->OW - p->W + p->KW - 1 - p->PW;
      int lower[3] = {-p->PW, -p->PH, -p->PT};
      int upper[3] = {ph_w - (p->KW - 1), ph_h - (p->KH - 1), ph_t - (p->KT - 1)};
      for (int i = 0; i < 3; ++i)
        STEP_CHECK_ARG(lower[i] >= -16 && lower[i] <= 15 && upper[i] >= -16 && upper[i] <= 15, "conv3d(f16): im2col corner range");
      rc = encode_act5d_im2col(&pl->map_a, p->x, act, lower, upper, BK, kBM, swizzle_for(BK),
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "conv3d(f16): A (im2col)");
      // Same work-around CUTLASS applies (cute/atom/copy_traits_sm90_im2col.hpp): drivers <= 13.1 set a
      // descriptor bit that breaks im2col loads from tensors smaller than 128 KiB.
      int drv = 0;
      cudaDriverGetVersion(&drv);
      if (rc == 0 && drv <= 13010 &&
          (size_t)p->N * p->T * p->H * p->W * p->in_ld * 2 < 131072)
        reinterpret_cast<uint64_t*>(&pl->map_a)[1] &= ~(1ULL << 21);
      m_tiles = (g.M + kBM - 1) / kBM;
      g.a_bytes = kBM * BK * 2;
    }
  }
  if (rc) return rc;
  if ((rc = encode_weights3d(&pl->map_b, p->w, p->Cout, taps, p->Cin, p->w_ld, BK, g.BN, swizzle_for(BK),
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "conv3d(f16): B")))
    return rc;
  STEP_CHECK_ARG(m_tiles * g.n_tiles < (1LL << 31), "conv3d(f16): grid too large");
  g.tiles = (int)(m_tiles * g.n_tiles);
  // Pipeline depth: at least three stages and the output staging tile within half of an SM's shared memory (<= 113 KB) when
  // the occupancy calculator says two such CTAs really fit an SM (registers included), so that one CTA's epilogue overlaps
  // the other's main loop (BK 64 / BN 64, a thin 1x1x1 layer bound by memory, ran 45 % slower as one 8-stage CTA per SM);
  // otherwise as deep as the 227 KB of one SM allow.
  const long per_stage = (long)kBM * BK * 2 + (long)g.BN * BK * 2;
  const long fixed = kBookBytes + 1024 + (long)kBM * staging_pitch(g.BN);
  int st = (int)((113L * 1024 - fixed) / per_stage);
  if (st > kStages) st = kStages;
  bool two = false;
  if (st >= 3) {
    if (int rc = two_ctas_fit(pl->tile, (size_t)(fixed + st * per_stage), &two)) return rc;
  }
  if (!two) st = (int)((227L * 1024 - fixed) / per_stage);
  g.n_stages = st > kStages ? kStages : st;
  STEP_CHECK_ARG(g.n_stages >= 2, "conv3d(f16): tile does not fit shared memory");
  pl->smem_bytes = (size_t)(fixed + g.n_stages * per_stage);
  // Persistent grid: as many CTAs as fit the device at once, each walking the tiles with a stride of the grid, in tile order
  // (the N tiles of one M tile run on neighbouring CTAs and share A in L2).  A tile with a K loop of more than
  // kPersistMaxKBlocks k-blocks already hides its fixed cost (prologue, pipeline fill, epilogue) behind its own MMAs, and the
  // hardware's dispatch of one tile per CTA to whichever SM frees first balances unequal tile times better than a fixed
  // stride: one CTA per tile there (Mixed 4e/4f/5b 3x3x3 at BK 32, 135 k-blocks, ran 6-12 % slower with the stride;
  // layers of up to 81 k-blocks run faster with it).
  int sms = 0;
  if (int rc = sm_count(&sms)) return rc;
  const long resident = (long)sms * (two ? 2 : 1);
  const bool persist = g.taps * g.kblocks_per_tap <= kPersistMaxKBlocks && g.tiles > resident;
  pl->grid = dim3((unsigned)(persist ? resident : g.tiles));
  return 0;
}

int conv3d_umma_launch(const step_conv_params* p, step_stream_t stream) {
  ConvPlan pl;
  if (int rc = build_plan(p, &pl)) return rc;
  const ConvTile& t = kTiles[pl.tile];
  if (int rc = allow_dynamic_smem(t.kernel, g_attr_seen[pl.tile], 227 * 1024, "conv_umma_kernel")) return rc;
  return launch_tc("conv_umma_kernel", t.kernel, pl.grid, kThreads, pl.smem_bytes, cu(stream), pl.map_a, pl.map_b, pl.g,
                   p->scale, p->shift, (const __half*)p->residual, (__half*)p->y);
}

}  // namespace step

using namespace step;

// Test hook (tests/test_gpu_conv.py): raw bytes of one staged A tile -> out [128 * BK * 2].
extern "C" int step_debug_tma_tile(const step_conv_params* p, int m_tile, int kt, int kh, int kw, int c0, void* out,
                                   int* bk_out, int* box_out /*[3]*/, step_stream_t stream) {
  ConvPlan pl;
  if (int rc = build_plan(p, &pl)) return rc;
  if (bk_out) *bk_out = pl.BK;
  if (box_out) { box_out[0] = pl.g.bw; box_out[1] = pl.g.bh; box_out[2] = pl.g.bt; }
  size_t smem = 1024 + (size_t)kBM * pl.BK * 2;
  if (pl.BK == 64) tma_dump_kernel<64><<<1, 32, smem, cu(stream)>>>(pl.map_a, pl.g, m_tile, kt, kh, kw, c0, (uint8_t*)out);
  else if (pl.BK == 32) tma_dump_kernel<32><<<1, 32, smem, cu(stream)>>>(pl.map_a, pl.g, m_tile, kt, kh, kw, c0, (uint8_t*)out);
  else tma_dump_kernel<16><<<1, 32, smem, cu(stream)>>>(pl.map_a, pl.g, m_tile, kt, kh, kw, c0, (uint8_t*)out);
  STEP_LAUNCH_CHECK("tma_dump_kernel");
  return 0;
}
