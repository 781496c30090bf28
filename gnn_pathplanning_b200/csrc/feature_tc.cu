// Tensor-core (wgmma, Hopper) feature extractor: the per-agent CNN + compress MLP of DecentralPlannerNet
// (reference graphs/models/decentralplanner.py:155-195,284-290, eval mode) as six implicit GEMMs per tile of up to
// 12 agents, fp32 parity through 3xTF32 split precision.
//
//   layer   GEMM rows per agent (M)          N (out ch)   K = taps x Cin   K chunks of 32
//   conv0   100 (10x10, 2x2-pool order)      32           27 (+5 zero)     1
//   conv1   25  (5x5)                        32           9 x 32           9   (chunk = tap)
//   conv2   16  (4x4, pool order)            64           9 x 32           9
//   conv3   4   (2x2)                        64           9 x 64           18  (chunk = tap, channel half)
//   conv4   4   (2x2, pool order)            128          9 x 64           18
//   linear  1                                128          128              4
//
// Activations live in shared memory channels-last (NHWC), so the im2col row of one tap is 128 contiguous
// bytes (or zeros outside the map): producers copy it, split it into tf32 hi/lo and store it in the
// canonical SWIZZLE_128B K-major layout.  Filters are pre-split / pre-swizzled chunk images streamed with
// cp.async.  Per layer the loop is M-tile outer, K-chunk inner: the MMA warpgroup (warps 8-11) keeps one
// 128-row accumulator in registers (two wgmma M = 64 halves), applies the folded BatchNorm + ReLU, max-pools
// across the 4 consecutive rows of a pooling window with warp shuffles and writes the next layer's NHWC input
// straight from its registers.
#include "common.cuh"
#include "feature.cuh"
#include "tc_common.cuh"

#include <stdlib.h>

namespace gpp {

constexpr int FT_THREADS = 256;            // producer threads (+ the MMA / epilogue warpgroup)
constexpr int FT_MMA_THREADS = 128;
constexpr int FT_AMAX = 12;                // agents per tile
constexpr int FT_OP_BYTES = 128 * 128;     // one operand half (hi or lo) of one A chunk: 16 KB
constexpr int FT_STAGE_BYTES = 2 * FT_OP_BYTES;
constexpr int FT_NS = 2;                   // ring depth; the A and B operands of an item share a slot
constexpr int FT_ACT_FLOATS = FT_AMAX * 800;          // one activation region: 25 positions x 32 channels per agent
constexpr int FT_IN0 = 3 * 144;                       // padded [3][12][12] input per agent
constexpr int FT_NLAYERS = 6;
// smem map (bytes from the 1024-aligned base)
constexpr int FT_OFF_A = 0;
constexpr int FT_OFF_B = FT_OFF_A + FT_NS * FT_STAGE_BYTES;
constexpr int FT_OFF_X = FT_OFF_B + FT_NS * FT_STAGE_BYTES;             // region X: act1 -> act3 -> act5
constexpr int FT_OFF_Y = FT_OFF_X + FT_ACT_FLOATS * 4;                  // region Y: in0  -> act2 -> act4
constexpr int FT_OFF_BAR = FT_OFF_Y + FT_ACT_FLOATS * 4;
constexpr int FT_SMEM_BYTES = FT_OFF_BAR + 256 + 1024;
static_assert(FT_AMAX * FT_IN0 <= FT_ACT_FLOATS, "padded inputs must fit region Y");

struct FtLayer {
    const float* img;    // B chunk images: per chunk { hi[N x 32] , lo[N x 32] } swizzled
    const float* sc;     // folded BatchNorm scale (null: 1)
    const float* sh;     // folded shift / bias
};
struct FtArgs {
    const float* x;
    float* feat;
    int total_agents, apt, num_tiles;
    FtLayer layer[FT_NLAYERS];
    unsigned long long* timing;    // optional [32] cycle counters (debug): per layer produce / wait / epilogue; [20..] fine
};

// compile-time layer table
__host__ __device__ constexpr int ft_n(int L) { return L < 2 ? 32 : (L < 4 ? 64 : 128); }
__host__ __device__ constexpr int ft_rows(int L) { return L == 0 ? 100 : L == 1 ? 25 : L == 2 ? 16 : L < 5 ? 4 : 1; }
__host__ __device__ constexpr int ft_nk(int L) { return L == 0 ? 1 : L < 3 ? 9 : L < 5 ? 18 : 4; }
__host__ __device__ constexpr int ft_pooled(int L) { return (L == 0 || L == 2 || L == 4) ? 1 : 0; }
__host__ __device__ constexpr int ft_wout(int L) { return L == 0 ? 10 : L == 1 ? 5 : L == 2 ? 4 : L < 5 ? 2 : 1; }
__host__ __device__ constexpr int ft_win(int L) { return L == 0 ? 11 : L < 3 ? 5 : L < 5 ? 2 : 1; }
__host__ __device__ constexpr int ft_cin(int L) { return L == 0 ? 3 : L < 3 ? 32 : L < 5 ? 64 : 128; }
// floats per agent of the NHWC output of layer L (after pooling)
__host__ __device__ constexpr int ft_out_stride(int L) { return L < 2 ? 800 : L < 4 ? 256 : 128; }

// One arrival per producer WARP (barrier count = 8) and one polling lane per warp: 256 threads arriving on /
// polling the same mbarrier serialise in the shared-memory atomic unit.
__device__ __forceinline__ void ft_mbar_arrive(uint64_t* bar) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0)
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ft_mbar_wait_warp(uint64_t* bar, uint32_t parity) {
    if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
    __syncwarp();
}
__device__ __forceinline__ void ft_producers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void ft_mma_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }

// (y, x) of GEMM row `idx` of one agent
template <int L>
__device__ __forceinline__ void ft_row_pos(int idx, int& y, int& x) {
    constexpr int W = ft_wout(L);
    if (ft_pooled(L)) {
        constexpr int HW = (W / 2 > 0) ? W / 2 : 1;
        const int pp = idx >> 2, w = idx & 3;
        y = 2 * (pp / HW) + (w >> 1);
        x = 2 * (pp % HW) + (w & 1);
    } else {
        y = idx / W;
        x = idx % W;
    }
}

// One layer, producer side: for every (M tile, k chunk) item stage the B chunk (cp.async) and the A chunk, then wait
// until the MMA warpgroup has written the layer's output (the next layer's input).
template <int L>
__device__ __forceinline__ void ft_produce_layer(const FtArgs& A, unsigned char* sm, const float* in_buf, int na,
                                                 uint64_t* full, uint64_t* done, uint64_t* layer_done, uint32_t& q,
                                                 uint32_t& nl, int tid, unsigned long long* fine) {
    constexpr int N = ft_n(L), ROWS = ft_rows(L), NK = ft_nk(L), CIN = ft_cin(L), WIN = ft_win(L);
    constexpr int B_BYTES = 2 * N * 128;                 // hi | lo chunk image
    const int ntiles = (na * ROWS + 127) >> 7;
    const int j = tid & 7;
    const char* img = reinterpret_cast<const char*>(A.layer[L].img);
    for (int mt = 0; mt < ntiles; ++mt) {
        for (int kc = 0; kc < NK; ++kc, ++q) {
            const int s = q % FT_NS;
            const long long f0 = clock64();
            if (q >= FT_NS) ft_mbar_wait_warp(&done[s], ((q / FT_NS) - 1) & 1);
            const long long f1 = clock64();
            {   // B chunk kc
                const uint32_t dst = smem_u32(sm + FT_OFF_B + s * FT_STAGE_BYTES);
                const char* src = img + (size_t)kc * B_BYTES;
                for (int u = tid; u < B_BYTES / 16; u += FT_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + u * 16), "l"(src + (size_t)u * 16)
                                 : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
            // tap / channel offset of this chunk
            int ky = 0, kx = 0, c0 = 0;
            if (L >= 1 && L <= 2) { ky = kc / 3; kx = kc % 3; }
            if (L >= 3 && L <= 4) { const int t = kc >> 1; ky = t / 3; kx = t % 3; c0 = (kc & 1) * 32; }
            if (L == 5) c0 = kc * 32;
            unsigned char* stage = sm + FT_OFF_A + s * FT_STAGE_BYTES;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = (tid >> 3) + 32 * i;
                const int m = mt * 128 + r;
                const int a = m / ROWS, idx = m - a * ROWS;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (a < na) {
                    int y, x;
                    ft_row_pos<L>(idx, y, x);
                    if (L == 0) {
                        // 27 = (c, ky, kx) window values out of the zero-bordered [3][12][12] input
                        const float* p0 = in_buf + a * FT_IN0 + y * 12 + x;
                        float e[4];
#pragma unroll
                        for (int qq = 0; qq < 4; ++qq) {
                            const int kk = j * 4 + qq;
                            const int c = kk / 9, rem = kk - c * 9;
                            e[qq] = (kk < 27) ? p0[c * 144 + (rem / 3) * 12 + (rem % 3)] : 0.f;
                        }
                        v = make_float4(e[0], e[1], e[2], e[3]);
                    } else {
                        const int iy = y + ky - 1, ix = x + kx - 1;
                        const bool ok = (L == 5) || (iy >= 0 && iy < WIN && ix >= 0 && ix < WIN);
                        if (ok) {
                            const int pos = (L == 5) ? 0 : (iy * WIN + ix);
                            v = ld_smem4(in_buf + a * (WIN * WIN * CIN) + pos * CIN + c0 + j * 4);
                        }
                    }
                }
                float4 hi, lo;
                split_tf32(v.x, hi.x, lo.x);
                split_tf32(v.y, hi.y, lo.y);
                split_tf32(v.z, hi.z, lo.z);
                split_tf32(v.w, hi.w, lo.w);
                const uint32_t off = sw128_offset(r, j);
                *reinterpret_cast<float4*>(stage + off) = hi;
                if (L != 0) *reinterpret_cast<float4*>(stage + FT_OP_BYTES + off) = lo;   // conv0 input is exact
            }
            const long long f2 = clock64();
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            fence_proxy_async_smem();
            const long long f3 = clock64();
            ft_mbar_arrive(&full[s]);
            const long long f4 = clock64();
            fine[0] += f1 - f0; fine[1] += f2 - f1; fine[2] += f3 - f2; fine[3] += f4 - f3; fine[4] += 1;
        }
    }
    ft_mbar_wait_warp(layer_done, nl & 1);
    ++nl;
}

// One layer, MMA warpgroup: per M tile the K chunks into a register accumulator, then BN/ReLU (-> 2x2 max-pool over
// 4 consecutive rows) -> NHWC activations / features.  Thread t holds rows 64 h + wg_row(t, i), columns wg_col(t, i).
template <int L>
__device__ __forceinline__ void ft_mma_layer(const FtArgs& A, unsigned char* sm, float* out_buf, int na, int a0,
                                             uint64_t* full, uint64_t* done, uint64_t* layer_done, uint32_t& q, int t,
                                             unsigned long long* fine) {
    constexpr int N = ft_n(L), ROWS = ft_rows(L), NK = ft_nk(L);
    const int ntiles = (na * ROWS + 127) >> 7;
    const float* sc = A.layer[L].sc;
    const float* sh = A.layer[L].sh;
    const int lane = t & 31;
    float acc[2][N / 2];
    for (int mt = 0; mt < ntiles; ++mt) {
        for (int kc = 0; kc < NK; ++kc, ++q) {
            const int s = q % FT_NS;
            const long long m0 = clock64();
            mbar_wait(&full[s], (q / FT_NS) & 1);
            const long long m1 = clock64();
            const uint32_t sa = smem_u32(sm + FT_OFF_A + s * FT_STAGE_BYTES);
            const uint32_t sb = smem_u32(sm + FT_OFF_B + s * FT_STAGE_BYTES);
            const uint64_t b_hi = gmma_desc_sw128(sb), b_lo = gmma_desc_sw128(sb + N * 128);
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint64_t a_hi = gmma_desc_sw128(sa + h * 8192), a_lo = gmma_desc_sw128(sa + FT_OP_BYTES + h * 8192);
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) wgmma_tf32<N>(acc[h], a_hi + 2 * ks, b_hi + 2 * ks, (kc | ks) != 0);
                if (L != 0) {
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) wgmma_tf32<N>(acc[h], a_lo + 2 * ks, b_hi + 2 * ks, 1u);
                }
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) wgmma_tf32<N>(acc[h], a_hi + 2 * ks, b_lo + 2 * ks, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            ft_mma_sync();
            if (t == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&done[s])) : "memory");
            fine[0] += m1 - m0; fine[1] += clock64() - m1;
        }
        // ---- epilogue of the M tile
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < N / 2; i += 2) {
                const int m = mt * 128 + 64 * h + wg_row(t, i), c = wg_col(t, i);
                const int a = m / ROWS, idx = m - a * ROWS;
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float sce = sc ? __ldg(sc + c + e) : 1.f;
                    float tt = fmaxf(fmaf(acc[h][i + e], sce, __ldg(sh + c + e)), 0.f);
                    if (ft_pooled(L)) {        // the 4 rows of a window are lanes 4 apart
                        tt = fmaxf(tt, __shfl_xor_sync(0xffffffffu, tt, 4));
                        tt = fmaxf(tt, __shfl_xor_sync(0xffffffffu, tt, 8));
                    }
                    v[e] = tt;
                }
                if (a < na && (!ft_pooled(L) || ((lane >> 2) & 3) == 0)) {
                    float* dst;
                    if (L == 5)
                        dst = A.feat + (size_t)(a0 + a) * 128 + c;
                    else
                        dst = out_buf + a * ft_out_stride(L) + (ft_pooled(L) ? (idx >> 2) : idx) * N + c;
                    *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
                }
            }
        }
    }
    ft_mma_sync();        // every thread's output stores are done
    if (t == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(layer_done)) : "memory");
}

__global__ void __launch_bounds__(FT_THREADS + FT_MMA_THREADS, 1) feature_tc_kernel(const FtArgs A) {
    extern __shared__ unsigned char smem_raw_ft[];
    const uint32_t raw = smem_u32(smem_raw_ft);
    unsigned char* sm = smem_raw_ft + (((raw + 1023u) & ~1023u) - raw);
    float* regX = reinterpret_cast<float*>(sm + FT_OFF_X);
    float* regY = reinterpret_cast<float*>(sm + FT_OFF_Y);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + FT_OFF_BAR);
    uint64_t* full = bars;                                   // [2] producers staged the item's A and B operands
    uint64_t* done = full + FT_NS;                           // [2] the MMAs of the item have completed
    uint64_t* layer_done = done + FT_NS;                     // [1] the layer's output is written
    const int tid = threadIdx.x, warp = tid >> 5;

    if (tid == 0) {
        for (int i = 0; i < FT_NS; ++i) { mbar_init(&full[i], FT_THREADS / 32); mbar_init(&done[i], 1); }
        mbar_init(layer_done, 1);
        fence_mbar_init();
    }
    __syncthreads();

    uint32_t q = 0;
    if (warp >= FT_THREADS / 32) {
        // ================= MMA + epilogue warpgroup =================
        const int t = tid - FT_THREADS;
        unsigned long long mfine[2] = {0, 0};
        for (int tile = blockIdx.x; tile < A.num_tiles; tile += gridDim.x) {
            const int a0 = tile * A.apt;
            const int na = min(A.apt, A.total_agents - a0);
            ft_mma_layer<0>(A, sm, regX, na, a0, full, done, layer_done, q, t, mfine);    // in0  -> act1 [a][25][32]
            ft_mma_layer<1>(A, sm, regY, na, a0, full, done, layer_done, q, t, mfine);    // act1 -> act2 [a][25][32]
            ft_mma_layer<2>(A, sm, regX, na, a0, full, done, layer_done, q, t, mfine);    // act2 -> act3 [a][4][64]
            ft_mma_layer<3>(A, sm, regY, na, a0, full, done, layer_done, q, t, mfine);    // act3 -> act4 [a][4][64]
            ft_mma_layer<4>(A, sm, regX, na, a0, full, done, layer_done, q, t, mfine);    // act4 -> act5 [a][128]
            ft_mma_layer<5>(A, sm, regY, na, a0, full, done, layer_done, q, t, mfine);    // act5 -> features (global)
        }
        if (A.timing && t == 0) { atomicAdd(&A.timing[26], mfine[0]); atomicAdd(&A.timing[27], mfine[1]); }
    } else {
        // ================= producers =================
        uint32_t nl = 0;        // layer_done phases consumed
        unsigned long long tacc[32];
        for (int i = 0; i < 32; ++i) tacc[i] = 0;
        for (int tile = blockIdx.x; tile < A.num_tiles; tile += gridDim.x) {
            const int a0 = tile * A.apt;
            const int na = min(A.apt, A.total_agents - a0);
            // stage the binary FOV tensors into the zero-bordered [3][12][12] layout (region Y; the previous tile's
            // last reader of region Y was layer 4, which completed before this thread's wait for layer 5 below)
            for (int i = tid; i < na * FT_IN0; i += FT_THREADS) {
                const int a = i / FT_IN0, rem = i - a * FT_IN0;
                const int c = rem / 144, p = rem - c * 144;
                const int yy = p / 12 - 1, xx = p % 12 - 1;
                float v = 0.f;
                if (yy >= 0 && yy < 11 && xx >= 0 && xx < 11)
                    v = __ldcg(A.x + (size_t)(a0 + a) * 363 + c * 121 + yy * 11 + xx);
                regY[i] = v;
            }
            ft_producers_sync();

#define FT_LAYER(Lx, IN)                                                                                      \
    {                                                                                                          \
        const long long t0 = clock64();                                                                        \
        ft_produce_layer<Lx>(A, sm, IN, na, full, done, layer_done, q, nl, tid, tacc + 20);                    \
        tacc[3 * Lx] += clock64() - t0;                                                                        \
    }

            FT_LAYER(0, regY)
            FT_LAYER(1, regX)
            FT_LAYER(2, regY)
            FT_LAYER(3, regX)
            FT_LAYER(4, regY)
            FT_LAYER(5, regX)
#undef FT_LAYER
            tacc[18] += 1;
        }
        if (A.timing && tid == 0)
            for (int i = 0; i < 26; ++i) atomicAdd(&A.timing[i], tacc[i]);
    }
}

// ---------------------------------------------------------------------------------------
// B chunk images of one layer.  w: [N][Cin][taps] (conv: taps = 9, torch [co][ci][ky][kx]; linear: taps = 1).
// K ordering: conv0 k = flat (c,ky,kx) padded to 32; Cin = 32: k = tap*32 + ci; Cin = 64: k = tap*64 + ci;
// linear: k = ci.  Chunk image = { hi[N x 32], lo[N x 32] }, SWIZZLE_128B K-major.
// ---------------------------------------------------------------------------------------
__global__ void prep_umma_conv_kernel(const float* __restrict__ w, float* __restrict__ img, int N, int Cin, int taps,
                                      int nk) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;     // (f, kc, kk)
    if (idx >= N * nk * 32) return;
    const int kk = idx & 31, kc = (idx >> 5) % nk, f = idx / (32 * nk);
    float val = 0.f;
    if (Cin == 3) {
        if (kk < 27) val = w[f * 27 + kk];
    } else if (taps == 1) {
        val = w[(size_t)f * Cin + kc * 32 + kk];
    } else {
        const int k = kc * 32 + kk, tap = k / Cin, ci = k - tap * Cin;
        val = w[((size_t)f * Cin + ci) * 9 + tap];
    }
    float hi, lo;
    split_tf32(val, hi, lo);
    float* base = img + (size_t)kc * (2 * N * 32);
    const uint32_t off = sw128_offset(f, kk >> 2) / 4 + (kk & 3);
    base[off] = hi;
    base[N * 32 + off] = lo;
}

static unsigned long long* g_ft_timing = nullptr;
int debug_feature_tc_timing(unsigned long long* out20) {
    if (!g_ft_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out20, g_ft_timing, 256, cudaMemcpyDeviceToHost);
    cudaMemset(g_ft_timing, 0, 256);
    return GPP_OK;
}

size_t feature_tc_image_floats(int L) { return (size_t)ft_nk(L) * 2 * ft_n(L) * 32; }

int launch_prep_feature_tc(const float* w, float* img, int L, cudaStream_t st) {
    const int N = ft_n(L), nk = ft_nk(L);
    const int n = N * nk * 32;
    prep_umma_conv_kernel<<<(n + 255) / 256, 256, 0, st>>>(w, img, N, ft_cin(L), L == 5 ? 1 : 9, nk);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

int launch_feature_tc_kernel(const FeArgs& fa, const float* const* imgs, cudaStream_t st) {
    FtArgs a;
    a.x = fa.x; a.feat = fa.feat; a.total_agents = fa.total_agents;
    for (int L = 0; L < FT_NLAYERS; ++L) {
        a.layer[L].img = imgs[L];
        a.layer[L].sc = (L < 5) ? fa.sc[L] : nullptr;
        a.layer[L].sh = (L < 5) ? fa.sh[L] : fa.b5;
    }
    // agents per tile: fill the SMs first, then grow the tile up to FT_AMAX (fewer filter re-reads)
    int apt = (fa.total_agents + sm_count() - 1) / sm_count();
    if (apt < 8) apt = fa.total_agents >= 8 ? 8 : fa.total_agents;
    if (apt > FT_AMAX) apt = FT_AMAX;
    a.apt = apt;
    a.num_tiles = (fa.total_agents + apt - 1) / apt;
    a.timing = nullptr;
    if (debug_option(DBG_TC_TIMING)) {
        if (!g_ft_timing) { cudaMalloc(&g_ft_timing, 256); cudaMemset(g_ft_timing, 0, 256); }
        a.timing = g_ft_timing;
    }
    static SmemConfig smem_cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(feature_tc_kernel, smem_cfg, FT_SMEM_BYTES));
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    feature_tc_kernel<<<grid, FT_THREADS + FT_MMA_THREADS, FT_SMEM_BYTES, st>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp
