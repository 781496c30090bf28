// Small-batch fused graph filter + action MLP on the Hopper tensor cores (wgmma; N = 10 agents, K <= 3 taps, planner
// path): the filter of the benchmark configuration (640 node rows), where the CUDA-core kernel's 10-row x 384 x 64
// contraction is latency- and shared-memory-bound.
//
//   y = ReLU(sum_k (x S^k) W_k + b),  logits = y Wa^T + ba          (reference: utils/graphUtils/graphML.py:2342-2366,
//                                                                    graphs/models/decentralplanner.py:221,301-318)
//
// One CTA = 6 samples (60 node rows, one M = 64 accumulator tile) x one 64-column half of the F = 128 outputs; the 2 CTAs
// of a tile are a thread-block cluster: the second one adds its partial logits into the first one's shared memory
// (st.shared::cluster) and a cluster barrier replaces the global-memory ticket of the CUDA-core kernel.  The CTA's half of the taps (fp16 hi | lo, no-swizzle
// K-major planes, 32 KB per tap) is fetched by bulk copies BEFORE the programmatic-launch wait, i.e. while the feature
// kernel still runs -- with 22 CTAs at the benchmark size they sit on SMs the feature kernel does not use.  After the
// wait: thread (sample, feature) reads its 10 node values, forms z_1 = x S and z_2 = z_1 S in registers, scales by the
// sample's power of two, splits into fp16 hi / lo and stores the K operand planes; warpgroup 0 issues K * 8 pairs of
// wgmma (A_hi x [W_hi | W_lo] with N = 128, A_lo x W_hi with N = 64, register accumulators), adds the three products,
// applies bias + ReLU and the 64-column part of the 5-wide action MLP straight from its registers.
#include "common.cuh"
#include "tc_common.cuh"

#include <cuda_fp16.h>
#include <stdio.h>

namespace gpp {

constexpr int GS_N = 10, GS_TS = 6;                                // 60 valid rows of the M = 64 tile
constexpr int GS_THREADS = 384;                                    // thread = (feature, samples s and s + 3)
constexpr int GS_SPT = GS_TS / (GS_THREADS / 128);                 // samples per thread
constexpr int GS_W_PLANE = 128 * 16;                               // one K plane of [W_hi | W_lo]: 128 rows x 16 B
constexpr int GS_Z_LBO = 64 * 16 + 16;                             // z planes padded by one row: conflict-free 2-byte stores

struct GsSmem {
    int w_off, zhi_off, zlo_off, s_off, wa_off, bias_off, part_off, misc_off, total;
    __host__ __device__ explicit GsSmem(int K) {
        int off = 0;
        w_off = off; off += K * 16 * GS_W_PLANE;
        zhi_off = off; off += K * 16 * GS_Z_LBO;
        zlo_off = off; off += K * 16 * GS_Z_LBO;
        s_off = off; off += GS_TS * GS_N * GS_N * 4;
        wa_off = off; off += 5 * 64 * 4;
        bias_off = off; off += 64 * 4;
        part_off = off; off += 2 * 64 * 8 * 4;          // this CTA's partial logits + the peer CTA's
        misc_off = off; off += 128;
        total = off;
    }
};

struct GsMisc {
    uint64_t w_full;
    uint32_t xmax[GS_TS];
    uint32_t colmax[GS_TS];
    float inv[GS_TS];
};

struct GsArgs {
    const float* x;          // [B][10][128] node-major
    const void* S;           // [B][10][10] f32 or f64
    const unsigned char* img;    // [2 halves][K*16 planes][128 (W_hi | W_lo rows)][8 halves]
    const float* cst;        // [0] = 2^-ew (inverse weight scale)
    const float* bias;       // [128]
    const float* wa;         // [5][128]
    const float* ba;         // [5]
    float* logits;           // [10][B][5]
    int B, K, num_tiles, s_is_f64, pdl;
};

// no-swizzle K-major operand: K planes `lbo` bytes apart, 8-row groups 128 bytes apart
__device__ __forceinline__ uint64_t gs_desc(uint32_t addr, uint32_t lbo) { return gmma_desc_nosw(addr, lbo, 128); }
__device__ __forceinline__ int gs_scale_exp(uint32_t bits) {       // m * 2^e in [2^9, 2^10)
    if (bits == 0) return 0;
    int e = 9 - ((int)(bits >> 23) - 127);
    return e < -110 ? -110 : (e > 110 ? 110 : e);
}
__device__ __forceinline__ float gs_pow2(int e) { return __int_as_float((e + 127) << 23); }
// watchdog: trap after ~1 s instead of hanging the GPU (no printf: a call would serialise the kernel's wgmma)
__device__ __forceinline__ void gs_wait(uint64_t* bar, uint32_t parity) {
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 2000000000LL) __trap();
}

template <int K>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GS_THREADS, 1) gf_small_mma_kernel(const GsArgs a) {
    extern __shared__ __align__(1024) unsigned char sm[];
    const GsSmem L(K);
    GsMisc* ms = reinterpret_cast<GsMisc*>(sm + L.misc_off);
    float* Ss = reinterpret_cast<float*>(sm + L.s_off);
    float* was = reinterpret_cast<float*>(sm + L.wa_off);
    float* biass = reinterpret_cast<float*>(sm + L.bias_off);
    float* part = reinterpret_cast<float*>(sm + L.part_off);
    const uint32_t sm_base = smem_u32(sm);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x >> 1, half = blockIdx.x & 1;
    const int b0 = tile * GS_TS, ns = min(GS_TS, a.B - b0);
    // ---- prologue: nothing here depends on the kernel in front of this one
    if (tid == 0) {
        mbar_init(&ms->w_full, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(&ms->w_full, (uint32_t)(K * 16 * GS_W_PLANE));
        const unsigned char* src = a.img + (size_t)half * K * 16 * GS_W_PLANE;
        for (int k = 0; k < K; ++k)
            bulk_g2s(sm + L.w_off + k * 16 * GS_W_PLANE, src + (size_t)k * 16 * GS_W_PLANE, 16 * GS_W_PLANE, &ms->w_full);
    }
    if (tid < GS_TS) { ms->xmax[tid] = 0; ms->colmax[tid] = 0; }
    for (int i = tid; i < 5 * 64; i += GS_THREADS) was[i] = __ldg(a.wa + (i >> 6) * 128 + half * 64 + (i & 63));
    if (tid < 64) biass[tid] = __ldg(a.bias + half * 64 + tid);
    const float inv_w = __ldg(a.cst);
    __syncthreads();
    griddep_launch_dependents();
    if (a.pdl) griddep_wait();           // x = the feature kernel's output

    // ---- operands: thread (sample s, feature f) for s = tid / 128 + 3 * u
    const int f = tid & 127;
    float xvs[GS_SPT][GS_N];
#pragma unroll
    for (int u = 0; u < GS_SPT; ++u) {
        const int s = (tid >> 7) + u * (GS_THREADS / 128);
        const bool live = s < ns;
        float* xv = xvs[u];
        float m = 0.f;
        const float* xp = a.x + ((size_t)(b0 + s) * GS_N) * 128 + f;
#pragma unroll
        for (int n = 0; n < GS_N; ++n) {
            xv[n] = live ? __ldcg(xp + n * 128) : 0.f;     // L2: written by the kernel this one may overlap (PDL)
            m = fmaxf(m, fabsf(xv[n]));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) atomicMax(&ms->xmax[s], __float_as_uint(m));
    }
    for (int i = tid; i < GS_TS * GS_N * GS_N; i += GS_THREADS) {
        const int sb = i / (GS_N * GS_N);
        float v = 0.f;
        if (sb < ns) {
            const size_t idx = (size_t)b0 * GS_N * GS_N + i;
            v = a.s_is_f64 ? (float)reinterpret_cast<const double*>(a.S)[idx] : reinterpret_cast<const float*>(a.S)[idx];
        }
        Ss[i] = v;
    }
    {
        if (K >= 2 && tid < GS_TS * GS_N) {       // largest absolute column sum of each sample's S (thread = one column)
            const int sb = tid / GS_N, n = tid - sb * GS_N;
            if (sb < ns) {
                const size_t idx = (size_t)(b0 + sb) * GS_N * GS_N + n;
                float cs = 0.f;
#pragma unroll
                for (int m = 0; m < GS_N; ++m)
                    cs += fabsf(a.s_is_f64 ? (float)reinterpret_cast<const double*>(a.S)[idx + m * GS_N]
                                           : reinterpret_cast<const float*>(a.S)[idx + m * GS_N]);
                atomicMax(&ms->colmax[sb], __float_as_uint(cs));
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < GS_SPT; ++u) {
        const int s = (tid >> 7) + u * (GS_THREADS / 128);
        const float* xv = xvs[u];
        // z_1 = x S, z_2 = z_1 S for this thread's feature, two output nodes per step (rows of S are read as 8-byte pairs)
        float z1[GS_N], z2[GS_N];
        const float colmax = __uint_as_float(ms->colmax[s]);
        const float* Sp = Ss + s * GS_N * GS_N;
        if (K >= 2) {
#pragma unroll
            for (int n = 0; n < GS_N; ++n) z1[n] = 0.f;
#pragma unroll
            for (int m = 0; m < GS_N; ++m) {
#pragma unroll
                for (int n = 0; n < GS_N; n += 2) {
                    const float2 sv = *reinterpret_cast<const float2*>(Sp + m * GS_N + n);
                    ffma2_s(xv[m], sv.x, sv.y, z1[n], z1[n + 1]);
                }
            }
        }
        if (K >= 3) {
#pragma unroll
            for (int n = 0; n < GS_N; ++n) z2[n] = 0.f;
#pragma unroll
            for (int m = 0; m < GS_N; ++m) {
#pragma unroll
                for (int n = 0; n < GS_N; n += 2) {
                    const float2 sv = *reinterpret_cast<const float2*>(Sp + m * GS_N + n);
                    ffma2_s(z1[m], sv.x, sv.y, z2[n], z2[n + 1]);
                }
            }
        }
        // |z_k| <= max|x| * max(1, colsum)^k: one power of two per sample
        const float g = fmaxf(1.f, colmax);
        const float bound = __uint_as_float(ms->xmax[s]) * (K >= 3 ? g * g : (K >= 2 ? g : 1.f));
        const int e = gs_scale_exp(__float_as_uint(bound));
        const float mul = gs_pow2(e);
        if (f == 0) ms->inv[s] = gs_pow2(-e) * inv_w;
        const uint32_t zrow = (uint32_t)((s * GS_N) * 16 + (f & 7) * 2);
        const uint32_t zp = (uint32_t)((f >> 3) * GS_Z_LBO);
#pragma unroll
        for (int k = 0; k < K; ++k) {
#pragma unroll
            for (int n = 0; n < GS_N; ++n) {
                const float v = (k == 0 ? xv[n] : (k == 1 ? z1[n] : z2[n])) * mul;
                const __half hi = __float2half_rn(v);
                const __half lo = __float2half_rn(v - __half2float(hi));
                const uint32_t off = (uint32_t)(k * 16 * GS_Z_LBO) + zp + zrow + (uint32_t)n * 16;
                *reinterpret_cast<__half*>(sm + L.zhi_off + off) = hi;
                *reinterpret_cast<__half*>(sm + L.zlo_off + off) = lo;
            }
        }
    }
    fence_proxy_async_smem();
    __syncthreads();
    // ---- MMAs (warpgroup 0): K * 8 steps of K = 16, accumulators acc [64 rows][W_hi cols 0..63 | W_lo cols 64..127]
    //      += A_hi x [W_hi | W_lo] and acc_lo [64 rows][64] += A_lo x W_hi (a separate accumulator: wgmma of different
    //      shapes on the same registers are not ordered)
    const int nrows = ns * GS_N;
    if (warp < 4) {
        float acc[64], acc_lo[32];
        gs_wait(&ms->w_full, 0);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < K * 8; ++j) {
            const uint64_t db = gs_desc(sm_base + L.w_off + 2 * j * GS_W_PLANE, GS_W_PLANE);
            wgmma_f16<128>(acc, gs_desc(sm_base + L.zhi_off + 2 * j * GS_Z_LBO, GS_Z_LBO), db, j > 0);
            wgmma_f16<64>(acc_lo, gs_desc(sm_base + L.zlo_off + 2 * j * GS_Z_LBO, GS_Z_LBO), db, j > 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        // ---- epilogue: element i (< 32) of this thread is (row, col) in acc and acc_lo, with its W_lo partner at acc[i + 32];
        //      the 4 lanes of a quad hold the 64 columns of the same two rows
        float p[2][5] = {{0.f, 0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f, 0.f}};
        const int r0 = wg_row(tid, 0);
        const float inv0 = ms->inv[min(r0 / GS_N, GS_TS - 1)], inv1 = ms->inv[min((r0 + 8) / GS_N, GS_TS - 1)];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int col = wg_col(tid, i), hr = (i >> 1) & 1;
            const float y = fmaxf(fmaf((acc[i] + acc_lo[i]) + acc[i + 32], hr ? inv1 : inv0, biass[col]), 0.f);
#pragma unroll
            for (int q5 = 0; q5 < 5; ++q5) p[hr][q5] = fmaf(y, was[q5 * 64 + col], p[hr][q5]);
        }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int q5 = 0; q5 < 5; ++q5) {
                p[hr][q5] += __shfl_xor_sync(0xffffffffu, p[hr][q5], 1);
                p[hr][q5] += __shfl_xor_sync(0xffffffffu, p[hr][q5], 2);
            }
        if ((lane & 3) == 0) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr)
                if (r0 + 8 * hr < nrows)
#pragma unroll
                    for (int q5 = 0; q5 < 5; ++q5) part[(r0 + 8 * hr) * 8 + q5] = p[hr][q5];
        }
    }
    __syncthreads();
    // ---- CTA 1 of the pair hands its partial logits to CTA 0 through distributed shared memory, CTA 0 adds the halves
    //      (half 0 first) and the action bias
    float* peer = part + 64 * 8;
    if (half == 1) {
        for (int i = tid; i < nrows * 5; i += GS_THREADS) {
            const int r = i / 5, q5 = i - r * 5;
            const float v = part[r * 8 + q5];
            asm volatile(
                "{\n\t.reg .b32 ra;\n\t"
                "mapa.shared::cluster.u32 ra, %0, 0;\n\t"
                "st.shared::cluster.f32 [ra], %1;\n\t}"
                ::"r"(smem_u32(peer + r * 8 + q5)), "f"(v) : "memory");
        }
    }
    cluster_sync_all();          // release / acquire at cluster scope: CTA 1's stores are visible to CTA 0
    if (half == 0) {
        for (int i = tid; i < nrows * 5; i += GS_THREADS) {
            const int r = i / 5, q5 = i - r * 5;
            const int b = b0 + r / GS_N, n = r % GS_N;
            a.logits[((size_t)n * a.B + b) * 5 + q5] =
                part[r * 8 + q5] + peer[r * 8 + q5] + __ldg(a.ba + q5);
        }
    }
}

// ---- weight images --------------------------------------------------------------------------------------------------
__global__ void gs_absmax_kernel(const float* __restrict__ w, int n, unsigned int* __restrict__ out) {
    float m = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}
// w: [F = 128][K][G = 128] (graphML.py:2437); image[half][plane p][n2 (128)][e]: reduction index kk = p * 8 + e = k * 128 + g,
// n2 < 64: W_hi of output f = half * 64 + n2, n2 >= 64: W_lo of output f = half * 64 + n2 - 64
__global__ void gs_prep_kernel(const float* __restrict__ w, __half* __restrict__ img, int K, const unsigned int* __restrict__ amax,
                               float* __restrict__ cst) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int per_half = K * 16 * 128 * 8;
    if (idx >= 2 * per_half) return;
    const int e = gs_scale_exp(*amax);
    if (idx == 0) cst[0] = gs_pow2(-e);
    const int half = idx / per_half;
    int r = idx - half * per_half;
    const int el = r & 7; r >>= 3;
    const int n2 = r & 127; r >>= 7;
    const int p = r;
    const int kk = p * 8 + el, k = kk >> 7, g = kk & 127;
    const int f = half * 64 + (n2 & 63);
    const float v = w[((size_t)f * K + k) * 128 + g] * gs_pow2(e);
    const __half hi = __float2half_rn(v);
    img[idx] = (n2 >= 64) ? __float2half_rn(v - __half2float(hi)) : hi;
}

size_t gf_small_arena_bytes(int K) { return (size_t)2 * K * 16 * GS_W_PLANE + 64; }
bool gf_small_supported(int N, int K) { return N == GS_N && K >= 1 && K <= 3; }

int launch_prep_gf_small(const float* w, float* arena, int K, cudaStream_t st) {
    unsigned char* base = reinterpret_cast<unsigned char*>(arena);
    float* cst = reinterpret_cast<float*>(base + (size_t)2 * K * 16 * GS_W_PLANE);
    unsigned int* amax = reinterpret_cast<unsigned int*>(cst + 4);
    GPP_CUDA_OK(cudaMemsetAsync(amax, 0, 4, st));
    gs_absmax_kernel<<<32, 256, 0, st>>>(w, 128 * K * 128, amax);
    GPP_LAUNCH_CHECK();
    const int n = 2 * K * 16 * 128 * 8;
    gs_prep_kernel<<<(n + 255) / 256, 256, 0, st>>>(w, reinterpret_cast<__half*>(base), K, amax, cst);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

template <int K>
static int gs_launch(const GsArgs& a, cudaStream_t st) {
    const GsSmem L(K);
    static SmemConfig cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(gf_small_mma_kernel<K>, cfg, (size_t)L.total));
    GPP_CUDA_OK(launch_maybe_pdl(gf_small_mma_kernel<K>, 2 * a.num_tiles, GS_THREADS, (size_t)L.total, st, a.pdl, a));
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

int launch_gf_forward_small(const float* x, const void* S, int s_is_f64, const float* arena, const float* bias,
                            const float* wa, const float* ba, float* logits, int B, int K, int pdl, cudaStream_t st) {
    GsArgs a;
    const unsigned char* base = reinterpret_cast<const unsigned char*>(arena);
    a.x = x; a.S = S; a.img = base; a.cst = reinterpret_cast<const float*>(base + (size_t)2 * K * 16 * GS_W_PLANE);
    a.bias = bias; a.wa = wa; a.ba = ba; a.logits = logits;
    a.B = B; a.K = K; a.num_tiles = (B + GS_TS - 1) / GS_TS; a.s_is_f64 = s_is_f64; a.pdl = pdl;
    if (K == 1) return gs_launch<1>(a, st);
    if (K == 2) return gs_launch<2>(a, st);
    return gs_launch<3>(a, st);
}

}  // namespace gpp
