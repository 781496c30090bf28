// Hopper (sm_90a) tensor-core helpers shared by the tensor-core kernels: wgmma with shared-memory operand descriptors,
// register accumulators, cluster and bulk-copy plumbing.
//
// Operand convention used throughout: K-major tiles in one of the two canonical shared-memory layouts that wgmma reads
// through a matrix descriptor --
//   * SWIZZLE_128B: rows of 128 bytes (32 tf32 or 64 fp16 values = one K chunk), 8-row groups of 1024 bytes, and inside
//     each row the 16-byte chunk j is stored at position j ^ (row & 7).  Tile bases are 1024-byte aligned.  One K step
//     (K = 8 tf32 or K = 16 fp16: 32 bytes) advances the descriptor's start address by 32 bytes inside the atom.
//   * no swizzle ("interleave"): 8 x 16-byte core matrices; rows 16 bytes apart, 8-row groups SBO bytes apart, the two
//     8-element K halves of a K = 16 step LBO bytes apart.
// A warpgroup (4 consecutive warps, the first one a multiple of 4) issues wgmma.mma_async for M = 64 rows; thread t of
// the warpgroup holds accumulator element i at row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2) and column
// 8 * (i / 4) + 2 * (t % 4) + i % 2 (wg_row / wg_col).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gpp {

// byte offset of (row, 16-byte chunk j) inside a SWIZZLE_128B K-major tile
__host__ __device__ __forceinline__ uint32_t sw128_offset(int row, int j) {
    return (uint32_t)(((row >> 3) << 10) + ((row & 7) << 7) + (((j ^ row) & 7) << 4));
}

// Shared-memory matrix descriptor (GMMA): start address >> 4 in bits [0,14), leading byte offset >> 4 in [16,30),
// stride byte offset >> 4 in [32,46), layout type in [62,64) (0 = no swizzle, 1 = SWIZZLE_128B).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint64_t gmma_desc_nosw(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

// Accumulator registers and shared-memory operands written by ordinary instructions must be ordered before the
// wgmma that reads them (the operand writers add fence.proxy.async before their barrier).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// accumulator element i of thread `t` (0..127 inside the warpgroup): row in [0, 64), column in [0, N)
__device__ __forceinline__ int wg_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int wg_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// D[64 x N] (+)= A[64 x K] . B[N x K]^T, fp32 accumulators d[N / 2]; accumulate = 0 overwrites d.
#define GPP_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                  "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_f16_n16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : GPP_D8(0) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_f16_n32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : GPP_D8(0), GPP_D8(8) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_f16_n64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : GPP_D8(0), GPP_D8(8), GPP_D8(16), GPP_D8(24) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_f16_n128(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : GPP_D8(0), GPP_D8(8), GPP_D8(16), GPP_D8(24), GPP_D8(32), GPP_D8(40), GPP_D8(48), GPP_D8(56) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                 : GPP_D8(0), GPP_D8(8) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                 : GPP_D8(0), GPP_D8(8), GPP_D8(16), GPP_D8(24) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
                 : GPP_D8(0), GPP_D8(8), GPP_D8(16), GPP_D8(24), GPP_D8(32), GPP_D8(40), GPP_D8(48), GPP_D8(56) : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
#undef GPP_D8

template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 16 || N == 32 || N == 64 || N == 128, "wgmma_f16: N");
    if constexpr (N == 16) wgmma_f16_n16(d, da, db, accumulate);
    else if constexpr (N == 32) wgmma_f16_n32(d, da, db, accumulate);
    else if constexpr (N == 64) wgmma_f16_n64(d, da, db, accumulate);
    else wgmma_f16_n128(d, da, db, accumulate);
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 32 || N == 64 || N == 128, "wgmma_tf32: N");
    if constexpr (N == 32) wgmma_tf32_n32(d, da, db, accumulate);
    else if constexpr (N == 64) wgmma_tf32_n64(d, da, db, accumulate);
    else wgmma_tf32_n128(d, da, db, accumulate);
}

// fp32 -> (hi, lo) with hi = tf32(x) (round to nearest), lo = tf32(x - hi): x = hi + lo up to 2^-22 |x|
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t h, l;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    const float rem = x - hi;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(rem));
    lo = __uint_as_float(l);
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

}  // namespace gpp
