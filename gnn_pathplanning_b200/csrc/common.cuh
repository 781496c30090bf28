// Shared helpers for libgnnpp_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>

#include "../../include/gnnpp_b200.h"

namespace gpp {

// ---- error plumbing -------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<unsigned long long> g_launches;

#define GPP_CUDA_OK(expr)                                                                  \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            ::gpp::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                             __FILE__, __LINE__);                                          \
            return GPP_ERR_CUDA;                                                           \
        }                                                                                  \
    } while (0)

#define GPP_REQUIRE(cond, code, ...)                                                       \
    do {                                                                                   \
        if (!(cond)) {                                                                     \
            ::gpp::set_error(__VA_ARGS__);                                                 \
            return code;                                                                   \
        }                                                                                  \
    } while (0)

#define GPP_LAUNCH_CHECK()                                                                 \
    do {                                                                                   \
        ::gpp::g_launches++;                                                               \
        GPP_CUDA_OK(cudaGetLastError());                                                   \
    } while (0)

int sm_count();       // SM count of the CURRENT device (cached per device ordinal)

// Debug switches (include/gnnpp_b200_debug.h: gpp_debug_set_option); all 0 in production.
enum DebugOption { DBG_GF_TIMING = 0, DBG_TC_TIMING = 1, DBG_FE_TIMING = 2, DBG_NO_PDL = 3, DBG_GF_MODE = 4, DBG_PAIR_ABLATE = 5, DBG_STAGE_MODE = 6, DBG_LANES = 7, DBG_COUNT = 8 };
int debug_option(int which);

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device function attribute: remember the largest
// value configured per device ordinal instead of one process-wide flag.
constexpr int kMaxDevices = 64;
struct SmemConfig {
    size_t bytes[kMaxDevices] = {};
};
template <typename Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kernel, SmemConfig& cfg, size_t smem) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < kMaxDevices && cfg.bytes[dev] >= smem) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess && dev >= 0 && dev < kMaxDevices) cfg.bytes[dev] = smem;
    return e;
}

// Launch with (pdl != 0) or without the programmatic-stream-serialization attribute.
template <typename Kernel, typename Args>
inline cudaError_t launch_maybe_pdl(Kernel kernel, int grid, int block, size_t smem, cudaStream_t st, int pdl,
                                    const Args& args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3((unsigned)block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, args);
}

// ---- device-side PTX helpers (mbarrier + 1-D bulk async copy, sm_90) -----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
                 : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy writes/reads of smem must be ordered before async-proxy (bulk copy) writes
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// ---- programmatic dependent launch: the next kernel of the stream may start its prologue early; its reads of
//      anything the previous kernels wrote come after griddep_wait() ------------------------------------------
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__device__ __forceinline__ float4 ld_smem4(const float* p) {
    return *reinterpret_cast<const float4*>(p);
}

// ---- paired fp32 arithmetic on two lanes of data with one scalar factor.  sm_90 has no packed fp32 instruction, so
//      these are two IEEE operations each (round to nearest, no contraction beyond the explicit fma). --------------
// (c0, c1) = s * (b0, b1) + (c0, c1)
__device__ __forceinline__ void ffma2_s(float s, float b0, float b1, float& c0, float& c1) {
    c0 = __fmaf_rn(s, b0, c0);
    c1 = __fmaf_rn(s, b1, c1);
}
// (c0, c1) = s * (b0, b1)
__device__ __forceinline__ void fmul2_s(float s, float b0, float b1, float& c0, float& c1) {
    c0 = __fmul_rn(s, b0);
    c1 = __fmul_rn(s, b1);
}
// (c0, c1) = (a0, a1) - (b0, b1)
__device__ __forceinline__ void fsub2(float a0, float a1, float b0, float b1, float& c0, float& c1) {
    c0 = __fsub_rn(a0, b0);
    c1 = __fsub_rn(a1, b1);
}

}  // namespace gpp
