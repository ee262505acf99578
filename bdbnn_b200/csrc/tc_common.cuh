// Shared wgmma / TMA / mbarrier PTX wrappers and tensor-map helpers (sm_90a).
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"

namespace bdbnn {

// ---------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
// Bounded spin: a protocol bug traps (launch error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  for (uint32_t spin = 0; !ok; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (spin > (1u << 24)) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, "
      "%5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// Thread-block clusters.  A CTA's rank in its cluster is x + y * (cluster width).
// Arrive on the barrier at the same shared-memory offset in cluster CTA `rank` (which may be this CTA).
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(bar), "r"(rank)
      : "memory");
}
// Every thread of every CTA of the cluster; also orders the CTA's own threads like __syncthreads.
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// TMA loads written to the same shared-memory offset of every cluster CTA in `mask` (bit = rank); each receiving
// CTA's barrier at offset `bar` gets the complete_tx of the bytes written into it.
__device__ __forceinline__ void tma_load_4d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                               int c2, int c3, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%3, %4, %5, %6}], [%2], %7;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                               uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}


// Warpgroup MMA (wgmma, sm_90a).  A warpgroup is four consecutive warps whose first warp index is a multiple of 4;
// all 128 threads issue each wgmma together and the accumulator lives in their registers.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads/writes across an in-flight wgmma.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (sm_90 GMMA layout): start address >> 4 in [0,14), LBO >> 4 in [16,30),
// SBO >> 4 in [32,46), layout type in [62,64) (1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B).
// K-major swizzled tiles: LBO unused, SBO = bytes between 8-row groups = 8 * row_bytes; a K step inside a
// swizzled row advances the start address by its byte width (the swizzle XOR is applied to address bits).
// MN-major swizzled tiles: LBO = bytes between swizzle-row-wide MN chunks, SBO = bytes between 8-row K groups.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t row_bytes) {
  const uint32_t layout = row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : 3u);
  uint64_t d = 0;
  d |= uint64_t((saddr & 0x3FFFFu) >> 4);
  d |= uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= uint64_t(((8u * row_bytes) >> 4) & 0x3FFFu) << 32;
  d |= uint64_t(layout) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr, uint32_t row_bytes) {
  return make_smem_desc(saddr, 16u, row_bytes);
}

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, fp32 accumulate in the warpgroup's registers (d: N/2 per thread).
// KIND 0: fp16, 1: bf16 (K = 16; TA/TB = 1 for MN-major operands), 2: fp8 e4m3 (K = 32, K-major only).
// Accumulator layout: thread t (warp w = t/32, lane l) holds rows 16w + l/4 (+8) and columns
// 8j + 2(l%4) (+1): d[4j + 0/1] = row 16w + l/4, d[4j + 2/3] = row 16w + l/4 + 8.
template <int N, int KIND, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db) {
  static_assert(N == 16 || N == 32 || N == 64 || N == 128 || (N == 256 && KIND != 2),
                "wgmma_ss: N in {16, 32, 64, 128}, or 256 with 16-bit operands");
  static_assert(KIND >= 0 && KIND <= 2, "wgmma_ss: KIND in {0, 1, 2}");
  if constexpr (N == 16 && KIND == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %10, %11;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 16 && KIND == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %10, %11;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 16 && KIND == 2) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db)
        : "memory");
  }
  if constexpr (N == 32 && KIND == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %18, %19;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 32 && KIND == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %18, %19;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 32 && KIND == 2) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db)
        : "memory");
  }
  if constexpr (N == 64 && KIND == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 64 && KIND == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 64 && KIND == 2) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db)
        : "memory");
  }
  if constexpr (N == 128 && KIND == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %67;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 128 && KIND == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %67;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 128 && KIND == 2) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db)
        : "memory");
  }
  if constexpr (N == 256 && KIND == 0) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %130, %131;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
  if constexpr (N == 256 && KIND == 1) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %130, %131;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "n"(TA), "n"(TB)
        : "memory");
  }
}

// Tensor-core kernels: warpgroups 0 and 1 issue the wgmmas for rows [0, 64) and [64, 128) of every 128-row
// M tile and run the epilogue from their registers; warp 8 (lane 0) is the TMA producer.
constexpr int kTcThreads = 288;
constexpr int kProducerWarp = 8;
constexpr int kMaxStages = 8;
constexpr int kTileM = 128;
constexpr int kMaxTaps = 49;

// ---------------------------------------------------------------------------------------------------
// Host side: tensor-map construction and launch
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

inline CUtensorMapSwizzle swizzle_for(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// bf16 NHWC activation tensor [N][H][W][C] -> 4-D map, box [BNI][BH][BW][KB].
// esize = 2: 16-bit elements (bf16/fp16 bit patterns), esize = 1: fp8 bytes.
inline int make_act_map(CUtensorMap* map, const void* base, int N, int H, int W, int C, int KB, int BW,
                        int BH, int BNI, int step = 1, int esize = 2) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return BDBNN_ERR_CUDA; }
  cuuint64_t dims[4] = {cuuint64_t(C), cuuint64_t(W), cuuint64_t(H), cuuint64_t(N)};
  cuuint64_t strides[3] = {cuuint64_t(C) * esize, cuuint64_t(W) * C * esize, cuuint64_t(H) * W * C * esize};
  // element stride `step` in w/h: TMA loads ceil(box/step) elements, so box = loaded * step
  cuuint32_t box[4] = {cuuint32_t(KB), cuuint32_t(BW * step), cuuint32_t(BH * step), cuuint32_t(BNI)};
  cuuint32_t estr[4] = {1, cuuint32_t(step), cuuint32_t(step), 1};
  CUresult r = enc(map, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_for(KB * esize),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(act) failed: %d", int(r)); return BDBNN_ERR_CUDA; }
  return BDBNN_OK;
}

// Overlapping-window view of a zero-padded 16-bit NHWC image (stem conv, stem.cu): element
// (j, wo, hp, n) lives at base + n*img_stride + hp*row_stride + wo*win_stride + 2*j (bytes), i.e. window
// `wo` of a padded row is the KB consecutive values starting win_stride bytes after window wo-1 —
// consecutive windows overlap; TMA only needs every stride to be a multiple of 16 bytes.
// Box [BNI][BH (every hstep-th row)][BW][KB].
inline int make_window_map(CUtensorMap* map, const void* base, int N, int HP, int WO, int KB,
                           uint64_t win_stride, uint64_t row_stride, uint64_t img_stride, int BW, int BH,
                           int BNI, int hstep) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return BDBNN_ERR_CUDA; }
  cuuint64_t dims[4] = {cuuint64_t(KB), cuuint64_t(WO), cuuint64_t(HP), cuuint64_t(N)};
  cuuint64_t strides[3] = {win_stride, row_stride, img_stride};
  cuuint32_t box[4] = {cuuint32_t(KB), cuuint32_t(BW), cuuint32_t(BH * hstep), cuuint32_t(BNI)};
  cuuint32_t estr[4] = {1, 1, cuuint32_t(hstep), 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(KB * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(window) failed: %d", int(r)); return BDBNN_ERR_CUDA; }
  return BDBNN_OK;
}

// bf16 K-major weight matrix [rows][cols] -> 2-D map, box [BN rows][KB cols].
inline int make_weight_map(CUtensorMap* map, const void* base, int rows, int cols, int KB, int BN, int esize = 2) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return BDBNN_ERR_CUDA; }
  cuuint64_t dims[2] = {cuuint64_t(cols), cuuint64_t(rows)};
  cuuint64_t strides[1] = {cuuint64_t(cols) * esize};
  cuuint32_t box[2] = {cuuint32_t(KB), cuuint32_t(BN)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_for(KB * esize),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weight) failed: %d", int(r)); return BDBNN_ERR_CUDA; }
  return BDBNN_OK;
}


// One implicit-GEMM launch: D[NIMG x OH x OW pixels, Nout] = sum_taps A[pixel*in_step + tap offset] * B.
struct TcConvLaunch {
  const uint16_t* A; int IH, IW, Kc, a_halves, in_step;
  const uint16_t* B; int b_taps, Nout;
  int NIMG, OH, OW;
  int n_taps; int8_t dh[kMaxTaps], dw[kMaxTaps]; uint8_t tb[kMaxTaps];
  int out_step, off_h, off_w, OHf, OWf;
  const float* alpha; const uint32_t* mask; float* out;
  int16_t* out_i16;              // forward, wide GEMMs only: write the integer accumulator as int16 instead of out
  int fmt;                       // operand format (BDBNN_FMT_*); -1 = fp8 e4m3 bytes (forward only)
  const uint32_t* amax_bits;     // FP16S gradient / real-valued eval operand: device word with max|A|; the
                                 // epilogue multiplies the accumulator by 2^-e
  const float* add;              // dgrad: optional tensor added to the result (shortcut gradient), or NULL;
                                 // eval: optional residual added to z
  // eval, 16-bit operands: pad_res = 1 reads the residual as the option-A shortcut add[n][2*oh][2*ow][c - res_coff]
  // of an NHWC [.][res_H][res_W][res_C] tensor, +0.0 outside the channel band (tc_conv_kernel's PADRES instances)
  int pad_res, res_H, res_W, res_C, res_coff;
  // eval forward (MODE 2): z = acc * alpha + shift (+ add) written to `out`, optional +-1 copies of z
  const float* shift; uint16_t* zb; uint8_t* zb8;
  int relu;                      // eval: z = relu(z) after the residual
  int hardtanh;                  // eval, fp16 operands, no option-A residual: z = clamp(z, -1, 1) instead of relu
  uint32_t* z_amax;              // eval: optional bits of max|z| (zeroed by the caller)
  // forward only: per-output-channel BatchNorm statistics of the result, accumulated by the epilogue
  // (sum y, sum y^2 as doubles [2*Nout]; max|y| bits [Nout]); NULL = off.  Zeroed by the caller.
  double* bn_sums;
  uint32_t* bn_ymax;
  // dgrad only (wide GEMMs, stride 1): bn_sums / bn_ymax receive the BACKWARD statistics of the BatchNorm
  // unit that produced this conv's input — sum gz, sum gz*yhat, max|gz| with gz = this launch's result — using
  // that unit's int16 conv result st_y [pixels][Nout] and per-channel alpha / mean / invstd
  const int16_t* st_y; const float* st_alpha; const float* st_mean; const float* st_invstd;
  // stem conv: A is an overlapping-window view (make_window_map) instead of a dense NHWC tensor
  int win;                       // 0 = dense NHWC
  uint64_t win_stride, win_row_stride, win_img_stride;
  // grouped conv as a banded GEMM (DESIGN.md §4t): band = B > 0 makes the N tile one band [n0, n0 + B) of Nout,
  // Kc = B, and the activation box's channel coordinate n0 + k over A's a_chans channels (tc_conv_kernel's BANDED
  // instances); 0 = dense
  int band, a_chans;
};

// Geometry of the stem's packed input (stem.cu): fp16 [N][HP][WP][4] zero-padded by 3 on every side,
// windows of 8 pixels (32 values) every 2 pixels.
struct StemGeom {
  int N, H, W, Ho, Wo, HP, WP;
  uint64_t win_stride, row_stride, img_stride;   // bytes
};
inline bool stem_geom(int N, int H, int W, StemGeom* g) {
  if (N < 1 || H < 7 || W < 7) return false;
  g->N = N; g->H = H; g->W = W;
  g->Ho = (H + 6 - 7) / 2 + 1; g->Wo = (W + 6 - 7) / 2 + 1;
  if (g->Wo > kTileM || g->Wo < 1) return false;
  g->HP = H + 6;
  int wp = W + 6 > 2 * g->Wo + 6 ? W + 6 : 2 * g->Wo + 6;
  g->WP = (wp + 7) & ~7;
  g->win_stride = 16;                               // 2 pixels x 4 halves x 2 bytes
  g->row_stride = uint64_t(g->WP) * 8;
  g->img_stride = g->row_stride * uint64_t(g->HP);
  return true;
}
constexpr int kStemCout = 64, kStemTaps = 7, kStemWin = 32;
int launch_stem_fwd(const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y, const StemGeom& g,
                    double* bn_sums, uint32_t* bn_ymax, cudaStream_t st);
int launch_stem_eval(const uint16_t* xw, const uint16_t* wf, const float* scale, const float* shift, float* z,
                     const StemGeom& g, int relu, uint32_t* z_amax, cudaStream_t st);
// zero the statistics buffers of a conv launch (no-op when off)
inline int bn_stats_zero(double* sums, uint32_t* ymax, int C, cudaStream_t st) {
  if (!sums) return BDBNN_OK;
  BDBNN_CUDA(cudaMemsetAsync(sums, 0, size_t(2 * C) * sizeof(double), st));
  BDBNN_CUDA(cudaMemsetAsync(ymax, 0, size_t(C) * sizeof(uint32_t), st));
  return BDBNN_OK;
}
size_t stem_wgrad_workspace_bytes(const StemGeom& g);
int launch_stem_wgrad(const uint16_t* gys, const uint16_t* xw, float* ws, size_t ws_bytes, int* ksplit_out,
                      const StemGeom& g, cudaStream_t st);

void set_tc_trace(long long* buf);
long long* get_tc_trace();
bool wgrad_tc_ok(const bdbnn_conv_shape* s);
// shapes of the binary tensor-core conv (b1_conv.cu, DESIGN.md §4x)
bool b1_shape_ok(const bdbnn_conv_shape* s);
// grouped 3x3 convs (DESIGN.md §4t): the band B of the banded kernels (0 = not supported), and whether the banded
// weight gradient has a plan
int gconv_band(const bdbnn_conv_shape* s, int groups);
bool gwgrad_tc_ok(const bdbnn_conv_shape* s, int band);

}  // namespace bdbnn
