// umma_ptx.cuh -- thin PTX wrappers shared by the tensor-core kernels (mbarrier, TMA loads / stores, wgmma descriptors and
// instructions), and their host side: tensor maps of the project's fp16 layouts and the launch.  sm_90a only.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <utility>

#include "common.cuh"

namespace step {

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over the `n` threads of the consumer warpgroups (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_im2col_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c, int w, int h,
                                                   int d, int n, uint16_t ow, uint16_t oh, uint16_t od) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2], {%8, %9, %10};"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(d), "r"(n), "h"(ow), "h"(oh), "h"(od) : "memory");
}
// bulk tensor store shared -> global (2-D map, coordinates {column, row}); out-of-range elements are not written
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
// bulk copy of `bytes` contiguous bytes shared -> global (both 16-byte aligned, bytes a multiple of 16)
__device__ __forceinline__ void bulk_store(void* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
// Four 8 x 8 fp16 matrices stored transposed: v[m] holds this thread's pair (row lane / 4, columns 2 (lane % 4) + {0, 1})
// of matrix m; lanes 8 m .. 8 m + 7 give the addresses of its memory rows 0..7, and memory row c receives column c.
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t* v) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest N committed bulk stores have finished reading their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor (PTX ISA, "Matrix Descriptor Format" for wgmma):
// [0,14) start >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4 | [62,64) swizzle
// (0 none, 1 = 128B, 2 = 64B, 3 = 32B).  K-major swizzled tiles as TMA writes them: rows of BK fp16, SBO = 8-row group pitch,
// LBO unused (1); advancing K by 16 elements inside the swizzle atom adds 32 bytes to the start address.
template <int BK>
__device__ __forceinline__ uint64_t desc_hi_kmajor() {
  constexpr uint64_t sw = BK == 64 ? 1 : (BK == 32 ? 2 : 3);
  return (1ULL << 16) | ((uint64_t)((8 * BK * 2) >> 4) << 32) | (sw << 62);
}
__device__ __forceinline__ uint64_t desc_lo(const void* p) { return (uint64_t)((smem_u32(p) & 0x3FFFF) >> 4); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 inputs, fp32 accumulator in N / 2 registers per thread of the warpgroup:
// d[4 j + 2 i + c] = row (warp % 4) * 16 + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + c, j < N / 8.  One instruction
// covers the whole N extent, so the 64 x 16 A slice is read from shared memory once per k16 step.  Defined for the N tile
// widths the kernels instantiate (conv_umma.cu STEP_CONV_TILES, and 64 for the patch and bottleneck-exit kernels); the
// accumulator operand list is spelled out per N because inline PTX takes only literal operand numbers.
template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t da, uint64_t db, uint32_t accumulate);

#define STEP_D4(i) "+f"(d[4 * (i)]), "+f"(d[4 * (i) + 1]), "+f"(d[4 * (i) + 2]), "+f"(d[4 * (i) + 3])
#define STEP_WGMMA_F16(N, IA, IB, IC, REGS, ...)                                                                        \
  template <>                                                                                                          \
  __device__ __forceinline__ void wgmma_f16<N>(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {              \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IC ", 0;\n\t"                                              \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, %" #IA ", %" #IB ", p, 1, 1, 0, 0;\n\t}" \
                 : __VA_ARGS__ : "l"(da), "l"(db), "r"(accumulate));                                                    \
  }
STEP_WGMMA_F16(32, 16, 17, 18,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3))
STEP_WGMMA_F16(64, 32, 33, 34,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7))
STEP_WGMMA_F16(128, 64, 65, 66,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15))
STEP_WGMMA_F16(144, 72, 73, 74,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17))
STEP_WGMMA_F16(152, 76, 77, 78,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18))
STEP_WGMMA_F16(160, 80, 81, 82,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19))
STEP_WGMMA_F16(176, 88, 89, 90,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21))
STEP_WGMMA_F16(192, 96, 97, 98,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21), STEP_D4(22), STEP_D4(23))
STEP_WGMMA_F16(208, 104, 105, 106,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21), STEP_D4(22), STEP_D4(23),
               STEP_D4(24), STEP_D4(25))
STEP_WGMMA_F16(224, 112, 113, 114,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, "
               "%105, %106, %107, %108, %109, %110, %111",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21), STEP_D4(22), STEP_D4(23),
               STEP_D4(24), STEP_D4(25), STEP_D4(26), STEP_D4(27))
STEP_WGMMA_F16(256, 128, 129, 130,
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, "
               "%105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, "
               "%122, %123, %124, %125, %126, %127",
               STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
               STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
               STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21), STEP_D4(22), STEP_D4(23),
               STEP_D4(24), STEP_D4(25), STEP_D4(26), STEP_D4(27), STEP_D4(28), STEP_D4(29), STEP_D4(30), STEP_D4(31))
#undef STEP_WGMMA_F16

// As wgmma_f16<N>, with A taken from registers: a[q] packs the fp16 pair of row (warp % 4) * 16 + lane / 4 + 8 (q & 1),
// columns 8 (q >> 1) + 2 (lane % 4) + {0, 1}.  That is the accumulator layout above, so accumulator registers
// [8 kk, 8 kk + 8) rounded pairwise to fp16 are the A operand of k-step kk.  Registers written by ordinary instructions
// need a wg_fence() before the first wgmma that reads them, and must not change until that wgmma has retired.
template <int N>
__device__ __forceinline__ void wgmma_f16_ra(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16_ra<256>(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
               "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
               "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
               "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, "
               "%65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, "
               "%86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, "
               "%105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, "
               "%122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
               : STEP_D4(0), STEP_D4(1), STEP_D4(2), STEP_D4(3), STEP_D4(4), STEP_D4(5), STEP_D4(6), STEP_D4(7),
                 STEP_D4(8), STEP_D4(9), STEP_D4(10), STEP_D4(11), STEP_D4(12), STEP_D4(13), STEP_D4(14), STEP_D4(15),
                 STEP_D4(16), STEP_D4(17), STEP_D4(18), STEP_D4(19), STEP_D4(20), STEP_D4(21), STEP_D4(22), STEP_D4(23),
                 STEP_D4(24), STEP_D4(25), STEP_D4(26), STEP_D4(27), STEP_D4(28), STEP_D4(29), STEP_D4(30), STEP_D4(31)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
#undef STEP_D4

__device__ __forceinline__ void wgmma_64x64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  wgmma_f16<64>(d, da, db, accumulate);
}

// Move registers between the warpgroups of a warp-specialised CTA (PTX setmaxnreg): every thread of the executing
// warpgroup must run it, and the CTA's total stays what it was launched with.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- host side ------------------------------------------------------------------------------
// The driver's tensor-map encoders, looked up once per process.  Function-local statics are initialised once even when
// several threads launch at the same time (nn.DataParallel replicas); a failed lookup stays null.
template <typename Fn>
inline Fn driver_entry_point(const char* symbol) {
  void* f = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPointByVersion(symbol, &f, 12000, cudaEnableDefault, &q) != cudaSuccess) f = nullptr;
  return (Fn)f;
}
inline PFN_cuTensorMapEncodeTiled_v12000 encode_tiled_fn() {
  static const auto fn = driver_entry_point<PFN_cuTensorMapEncodeTiled_v12000>("cuTensorMapEncodeTiled");
  return fn;
}
inline PFN_cuTensorMapEncodeIm2col_v12000 encode_im2col_fn() {
  static const auto fn = driver_entry_point<PFN_cuTensorMapEncodeIm2col_v12000>("cuTensorMapEncodeIm2col");
  return fn;
}

// TMA swizzle of a K-major tile with rows of BK fp16: the one desc_hi_kmajor<BK> describes to wgmma
inline CUtensorMapSwizzle swizzle_for(int BK) {
  return BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (BK == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// Every map below is fp16, element strides 1, no interleave, and loads zero-fill outside the tensor (OOB_FILL_NONE).
// Failures return STEP_E_DRIVER with `label` and the CUresult in the error text.
constexpr cuuint32_t kTmaOnes[5] = {1, 1, 1, 1, 1};

inline int encode_result(CUresult cr, const char* label) {
  if (cr != CUDA_SUCCESS) return fail(STEP_E_DRIVER, "%s: tensor map encode failed: CUresult %d", label, (int)cr);
  return 0;
}

inline int encode_tiled_f16(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                            const cuuint32_t* box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2,
                            const char* label) {
  const PFN_cuTensorMapEncodeTiled_v12000 enc = encode_tiled_fn();
  if (!enc) return fail(STEP_E_DRIVER, "cuTensorMapEncodeTiled entry point unavailable");
  return encode_result(enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides,
                           box, kTmaOnes, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
                       label);
}

// fp16 channels-last activation [N, T, H, W, ld], C live channels per pixel: the 5-D map {C, W, H, T, N}
struct ActLayout {
  cuuint64_t dims[5], strides[4];
  ActLayout(int N, int T, int H, int W, int C, int ld)
      : dims{(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)T, (cuuint64_t)N},
        strides{(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2, (cuuint64_t)T * H * W * ld * 2} {}
};

inline int encode_act5d(CUtensorMap* map, const void* x, const ActLayout& a, const cuuint32_t (&box)[5],
                        CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* label) {
  return encode_tiled_f16(map, x, 5, a.dims, a.strides, box, swizzle, l2, label);
}

// The same activation in TMA im2col mode: `channels` x `pixels` boxes walking the output pixels inside the bounding box
// [lower, upper] (w, h, t) of the padded input.
inline int encode_act5d_im2col(CUtensorMap* map, const void* x, const ActLayout& a, const int (&lower)[3],
                               const int (&upper)[3], int channels, int pixels, CUtensorMapSwizzle swizzle,
                               CUtensorMapL2promotion l2, const char* label) {
  const PFN_cuTensorMapEncodeIm2col_v12000 enc = encode_im2col_fn();
  if (!enc) return fail(STEP_E_DRIVER, "cuTensorMapEncodeIm2col entry point unavailable");
  return encode_result(enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(x), a.dims, a.strides, lower, upper,
                           (cuuint32_t)channels, (cuuint32_t)pixels, kTmaOnes, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
                       label);
}

// packed weights [Cout, taps, w_ld], Cin live channels per tap: the 3-D map {Cin, taps, Cout}, boxes of box_c channels
// of one tap for box_n output channels
inline int encode_weights3d(CUtensorMap* map, const void* w, int Cout, int taps, int Cin, int w_ld, int box_c, int box_n,
                            CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* label) {
  const cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)taps, (cuuint64_t)Cout};
  const cuuint64_t strides[2] = {(cuuint64_t)w_ld * 2, (cuuint64_t)taps * w_ld * 2};
  const cuuint32_t box[3] = {(cuuint32_t)box_c, 1, (cuuint32_t)box_n};
  return encode_tiled_f16(map, w, 3, dims, strides, box, swizzle, l2, label);
}

// row matrix [rows, cols] with a pitch of ld elements: the 2-D map {cols, rows}, boxes of box_c columns x box_r rows
inline int encode_rows2d(CUtensorMap* map, const void* base, long long rows, int cols, long long ld, int box_c, int box_r,
                         CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* label) {
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_c, (cuuint32_t)box_r};
  return encode_tiled_f16(map, base, 2, dims, strides, box, swizzle, l2, label);
}

// Launch of a TMA + wgmma kernel: launch errors reported naming the kernel, and the launch counted.
template <typename... Params, typename... Args>
inline int launch_tc(const char* name, void (*kernel)(Params...), dim3 grid, int threads, size_t smem, cudaStream_t stream,
                     Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) { cudaGetLastError(); return fail((int)e, "%s launch: %s", name, cudaGetErrorString(e)); }
  STEP_LAUNCH_CHECK(name);
  return 0;
}

}  // namespace step
