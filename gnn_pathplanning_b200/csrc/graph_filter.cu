// Fused K-tap graph filter for sm_90a (forward + backward).
//
// Replaces BatchLSIGF (gnn_pathplanning/utils/graphUtils/graphML.py:2273-2367):
//     z_0 = x,  z_k = z_{k-1} . S_b,   y[b,f,n] = sum_{k,g} w[f,0,k,g] z_k[b,g,n] + bias[f]
// One CTA owns a tile of TS whole samples (R = TS*N node rows):
//   1. the x rows and the dense GSO tile are staged into shared memory with 1-D bulk
//      async copies (cp.async.bulk -> UBLKCP) completing on an mbarrier,
//   2. the K-1 propagations z_k = S^T z_{k-1} run out of shared memory (node-major rows),
//   3. the tap contraction [R, K*G] x [K*G, F] streams the k-major taps from L2 with
//      coalesced register-double-buffered loads, 16 rows per register tile,
//   4. bias / ReLU / (optionally) the 128->5 action MLP with a warp-shuffle reduction run
//      in the epilogue; y is written once.
// fp32 FMA throughout: the result is within a few ulp of the reference's f32 matmuls.
#include "common.cuh"

#include <stdlib.h>

namespace gpp {

constexpr int GF_THREADS = 256;
constexpr int GF_WARPS = GF_THREADS / 32;
constexpr int GF_C = 128;        // G = F = 128 fast path
constexpr int GF_PS = GF_C + 4;  // padded row stride of a 128-wide smem tile
constexpr int GF_MAX_ROWS = 64;  // node rows per tile on the fast path
constexpr int NUM_ACT = 5;

// ---------------------------------------------------------------------------------------
// out[r][c] = sum_j in[r][j] * wm[j*ldw + c]   r < RP (mult of 16), c < n_out (mult of 32)
// A warp item is a 16-row x 32-column tile over one slice of the j range.  Shared memory returns 4 B per
// lane per clock while the FMA pipes take 4 operands per lane per clock, so every float read from shared
// memory has to feed >= 4 FMAs: each lane owns a 16 x 4 register tile (the 8 lanes of a quarter-warp cover
// the 32 columns, weights as one 16-byte load per row of wm), the 4 quarter-warps take every 4th group of
// 4 j's and meet through two shuffles per accumulator.  The rows of `in` are read as quarter-warp-uniform
// LDS.128 (a 128-bit load is served one quarter-warp at a time, so 4 addresses per instruction are free).
// nks > 1 splits the j range over items; slice ks writes its partial sums to out + ks*part_stride.
// Needs (n_in / nks) % 16 == 0, ldw % 4 == 0 and 16-byte aligned wm / in / out rows.
// WS: the weights are in shared memory, slice ks of the reduction range guarded by mbarrier wbar[ks]
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    return v;
}

template <bool WS>
__device__ __forceinline__ void tile_contract(const float* __restrict__ in_s, int IS, int n_in,
                                              const float* __restrict__ wm, int ldw, int n_out,
                                              float* __restrict__ out_s, int OS, int part_stride,
                                              int RP, int nks, uint64_t* wbar = nullptr) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int qw = lane >> 3, l8 = lane & 7;
    const int n_cg = n_out >> 5, n_rt = RP >> 4;
    const int n_items = n_cg * n_rt * nks;
    const int len = n_in / nks;
    for (int item = warp; item < n_items; item += nwarps) {
        const int cg = item % n_cg;
        const int rt = (item / n_cg) % n_rt;
        const int ks = item / (n_cg * n_rt);
        const int c4 = (cg << 5) + l8 * 4;
        const float* wp = wm + (size_t)(ks * len + qw * 4) * ldw + c4;
        const float* zr = in_s + (rt << 4) * IS + ks * len + qw * 4;
        float acc[16][4];
#pragma unroll
        for (int r = 0; r < 16; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
        if (WS) mbar_wait(wbar + ks, 0);
        float4 wn[4];
        if (!WS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) wn[j] = __ldg(reinterpret_cast<const float4*>(wp + (size_t)j * ldw));
        }
        for (int kb = 0; kb < len; kb += 16) {
            float4 w[4];
            if (WS) {
#pragma unroll
                for (int j = 0; j < 4; ++j) w[j] = ld_smem4(wp + (kb + j) * ldw);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) w[j] = wn[j];
                if (kb + 16 < len) {     // next block's filter rows are in flight while this one is used
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        wn[j] = __ldg(reinterpret_cast<const float4*>(wp + (size_t)(kb + 16 + j) * ldw));
                }
            }
#pragma unroll
            for (int r = 0; r < 16; r += 4) {
                float4 a[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = ld_smem4(zr + (r + i) * IS + kb);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float av[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        acc[r + i][0] = fmaf(av[j], w[j].x, acc[r + i][0]);
                        acc[r + i][1] = fmaf(av[j], w[j].y, acc[r + i][1]);
                        acc[r + i][2] = fmaf(av[j], w[j].z, acc[r + i][2]);
                        acc[r + i][3] = fmaf(av[j], w[j].w, acc[r + i][3]);
                    }
                }
            }
        }
        float* op = out_s + ks * part_stride + (rt << 4) * OS + c4;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            float4 v;
            v.x = quad_sum(acc[r][0]);
            v.y = quad_sum(acc[r][1]);
            v.z = quad_sum(acc[r][2]);
            v.w = quad_sum(acc[r][3]);
            if ((r & 3) == qw) *reinterpret_cast<float4*>(op + r * OS) = v;
        }
    }
}

// Stages the [ns, N, N] GSO tile into smem as f32 (plain path: any alignment, f32 or f64).
__device__ __forceinline__ void load_gso_plain(float* Ss, const void* S, int s_is_f64, size_t off,
                                               int count) {
    if (s_is_f64) {
        const double* Sd = reinterpret_cast<const double*>(S) + off;
        for (int i = threadIdx.x; i < count; i += blockDim.x) Ss[i] = static_cast<float>(Sd[i]);
    } else {
        const float* Sf = reinterpret_cast<const float*>(S) + off;
        for (int i = threadIdx.x; i < count; i += blockDim.x) Ss[i] = Sf[i];
    }
}

struct GfFwdArgs {
    const float* x;
    const void* S;
    const float* wt;      // [K*128][128] k-major taps
    const float* wsplit;  // [2][K*128][64] the same, column halves contiguous (w_smem launches)
    const float* bias;    // [128] or null
    float* y;             // null: do not write y
    const float* wa;      // [5][128] action weights, null: no fused action MLP
    const float* ba;      // [5]
    float* logits;        // [N][B][5]
    float* lpart;         // [csplit][B*N][5] partial logits (column-split launches only)
    unsigned int* tickets;  // [num_tiles] arrival counters of the column halves (zero before and after a launch)
    unsigned long long* timing;  // optional [8] per-phase cycle totals of block 0 (debug), null in production
    int B, N, K, TS, num_tiles, csplit;
    int s_is_f64, x_layout, y_layout, relu, bulk_x, bulk_s;
    int w_smem;           // column-split launch with one tile per CTA: this CTA's half of the taps is staged in smem
    int pdl;              // launched with programmatic stream serialization: wait before touching x
};

// smem carve-up shared by host (size) and device (pointers)
struct GfFwdSmem {
    int RP, ZS, nks, PS, s_floats, w_floats;
    __host__ __device__ GfFwdSmem(int N, int K, int TS, int csplit, int w_smem) {
        w_floats = w_smem ? K * GF_C * (GF_C / 2) : 0;
        RP = ((TS * N + 15) / 16) * 16;
        ZS = K * GF_C + 4;
        // split the K*G reduction so that the (4 / csplit) column groups x row tiles x splits fill 16 warps
        const int n_rt = RP / 16;
        nks = (n_rt >= 4 && (n_rt & 3) == 0) ? 1 : ((n_rt & 1) ? 4 : 2);
        nks *= csplit;
        if (nks > 8) nks = 8;
        PS = GF_C / csplit + 4;
        s_floats = ((TS * N * N + 3) / 4) * 4;
    }
    __host__ __device__ size_t z_off() const { return 96; }   // [0] staging barrier, [16..80) tap-slice barriers
    __host__ __device__ size_t s_off() const { return z_off() + sizeof(float) * RP * ZS; }
    __host__ __device__ size_t part_off() const { return s_off() + sizeof(float) * s_floats; }
    __host__ __device__ size_t misc_off() const {
        return part_off() + sizeof(float) * nks * RP * PS;
    }
    __host__ __device__ size_t w_off() const { return misc_off() + sizeof(float) * (GF_C + NUM_ACT * GF_C + 8); }
    __host__ __device__ size_t total() const { return w_off() + sizeof(float) * w_floats; }
};

constexpr int GF_FWD_THREADS = 512;
constexpr int GF_FWD_WARPS = GF_FWD_THREADS / 32;

__global__ void __launch_bounds__(GF_FWD_THREADS, 1) gf_fwd_kernel(const GfFwdArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const GfFwdSmem L(a.N, a.K, a.TS, a.csplit, a.w_smem);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
    uint64_t* wbar = reinterpret_cast<uint64_t*>(smem_raw + 16);
    float* wts = reinterpret_cast<float*>(smem_raw + L.w_off());
    __shared__ unsigned int s_last;
    float* z = reinterpret_cast<float*>(smem_raw + L.z_off());
    float* Ss = reinterpret_cast<float*>(smem_raw + L.s_off());
    float* part = reinterpret_cast<float*>(smem_raw + L.part_off());
    float* bias_s = reinterpret_cast<float*>(smem_raw + L.misc_off());
    float* wa_s = bias_s + GF_C;
    float* ba_s = wa_s + NUM_ACT * GF_C;
    const int N = a.N, K = a.K, ZS = L.ZS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool timed = a.timing && blockIdx.x == 0 && threadIdx.x == 0;
    long long tprev = timed ? clock64() : 0;
#define GF_MARK(i)                                                          \
    if (timed) {                                                            \
        const long long tn = clock64();                                     \
        atomicAdd(&a.timing[i], (unsigned long long)(tn - tprev));          \
        tprev = tn;                                                         \
    }

    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        if (a.w_smem) {
            // the taps do not depend on the previous kernel: their copy is in flight while x / S are staged and
            // propagated; one barrier per slice of the reduction range so that warps start as their slice lands
            const int len = a.K * GF_C / L.nks;
            const uint32_t bytes = (uint32_t)len * (GF_C / 2) * 4u;
            for (int ks = 0; ks < L.nks; ++ks) mbar_init(wbar + ks, 1);
            fence_mbar_init();
            const float* src = a.wsplit + (size_t)(blockIdx.x % a.csplit) * a.K * GF_C * (GF_C / 2);
            for (int ks = 0; ks < L.nks; ++ks) {
                mbar_arrive_expect_tx(wbar + ks, bytes);
                bulk_g2s(wts + (size_t)ks * len * (GF_C / 2), src + (size_t)ks * len * (GF_C / 2), bytes, wbar + ks);
            }
        } else {
            fence_mbar_init();
        }
    }
    for (int i = threadIdx.x; i < GF_C; i += GF_FWD_THREADS) bias_s[i] = a.bias ? a.bias[i] : 0.f;
    if (a.wa) {
        for (int i = threadIdx.x; i < NUM_ACT * GF_C; i += GF_FWD_THREADS) wa_s[i] = a.wa[i];
        if (threadIdx.x < NUM_ACT) ba_s[threadIdx.x] = a.ba[threadIdx.x];
    }
    __syncthreads();
    if (a.pdl) {
        griddep_wait();                 // x (the feature kernel's output) is complete and visible from here on
        griddep_launch_dependents();
    }
    GF_MARK(0)
    uint32_t phase = 0;

    // Column split (small batches): csplit CTAs share a tile, each contracts 128 / csplit output columns (half the
    // tap stream, half the dependent chain); the partial action logits meet in global memory and the CTA that
    // arrives last (ticket counter) adds them in a fixed order.
    const int ncols = GF_C / a.csplit;
    for (int vt = blockIdx.x; vt < a.num_tiles * a.csplit; vt += gridDim.x) {
        const int tile = vt / a.csplit, half = vt - tile * a.csplit;
        const int col0 = half * ncols;
        const int s0 = tile * a.TS;
        const int ns = min(a.TS, a.B - s0);
        const int R = ns * N;
        const int RP = ((R + 15) >> 4) << 4;
        const size_t row0 = (size_t)s0 * N;

        // ---- 1. stage x rows (k = 0 slot of z) and the GSO tile --------------------------
        if (a.bulk_x || a.bulk_s) {
            fence_proxy_async_smem();  // earlier generic-proxy traffic on z / Ss is done (synced)
            if (warp == 0) {
                if (lane == 0) {
                    uint32_t bytes = 0;
                    if (a.bulk_x) bytes += (uint32_t)R * GF_C * 4u;
                    if (a.bulk_s) bytes += (uint32_t)ns * N * N * 4u;
                    mbar_arrive_expect_tx(bar, bytes);
                    if (a.bulk_s)
                        bulk_g2s(Ss, reinterpret_cast<const float*>(a.S) + (size_t)s0 * N * N,
                                 (uint32_t)ns * N * N * 4u, bar);
                }
                __syncwarp();
                if (a.bulk_x)
                    for (int r = lane; r < R; r += 32)
                        bulk_g2s(z + r * ZS, a.x + (row0 + r) * GF_C, GF_C * 4u, bar);
            }
        }
        if (!a.bulk_s) load_gso_plain(Ss, a.S, a.s_is_f64, (size_t)s0 * N * N, ns * N * N);
        if (!a.bulk_x) {
            if (a.x_layout == GPP_NODE_MAJOR) {
                const float4* xp = reinterpret_cast<const float4*>(a.x + row0 * GF_C);
                for (int i = threadIdx.x; i < R * (GF_C / 4); i += GF_FWD_THREADS) {
                    const int r = i >> 5, q = i & 31;
                    *reinterpret_cast<float4*>(z + r * ZS + q * 4) = xp[i];
                }
            } else {  // [B, G, N]: contiguous per sample, transposed into node-major rows
                const float* xp = a.x + (size_t)s0 * GF_C * N;
                const int per = GF_C * N;
                for (int i = threadIdx.x; i < ns * per; i += GF_FWD_THREADS) {
                    const int bl = i / per, rem = i - bl * per;
                    const int g = rem / N, n = rem - g * N;
                    z[(bl * N + n) * ZS + g] = xp[i];
                }
            }
        }
        // zero the padding rows of the k = 0 slot (the other slots are produced below)
        for (int i = threadIdx.x; i < (RP - R) * GF_C; i += GF_FWD_THREADS)
            z[(R + i / GF_C) * ZS + (i % GF_C)] = 0.f;
        if (a.bulk_x || a.bulk_s) {
            mbar_wait(bar, phase);
            phase ^= 1;
        }
        __syncthreads();
        GF_MARK(1)

        // ---- 2. propagate: z_k[n,:] = sum_m S[m,n] z_{k-1}[m,:]  (x.S of graphML.py:2350) ---
        for (int k = 1; k < K; ++k) {
            for (int r = warp; r < RP; r += GF_FWD_WARPS) {
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                if (r < R) {
                    const int bl = r / N, n = r - bl * N;
                    const float* sp = Ss + bl * N * N + n;
                    const float* zp = z + (bl * N) * ZS + (k - 1) * GF_C + lane * 4;
                    for (int m = 0; m < N; ++m) {
                        const float s = sp[m * N];
                        const float4 v = ld_smem4(zp + m * ZS);
                        acc.x = fmaf(s, v.x, acc.x);
                        acc.y = fmaf(s, v.y, acc.y);
                        acc.z = fmaf(s, v.z, acc.z);
                        acc.w = fmaf(s, v.w, acc.w);
                    }
                }
                *reinterpret_cast<float4*>(z + r * ZS + k * GF_C + lane * 4) = acc;
            }
            __syncthreads();
        }

        GF_MARK(2)
        // ---- 3. tap contraction ---------------------------------------------------------
        const int nks = L.nks;  // fixed per launch: the partial buffers are sized for it
        if (a.w_smem)
            tile_contract<true>(z, ZS, K * GF_C, wts, GF_C / 2, ncols, part, L.PS, L.RP * L.PS, RP, nks, wbar);
        else
            tile_contract<false>(z, ZS, K * GF_C, a.wt + col0, GF_C, ncols, part, L.PS, L.RP * L.PS, RP, nks);
        __syncthreads();
        GF_MARK(3)

        // ---- 4. epilogue: bias, ReLU, y store, fused action MLP -------------------------
        for (int i = threadIdx.x; i < R * ncols; i += GF_FWD_THREADS) {
            const int r = i / ncols, f = i - r * ncols;
            float v = part[r * L.PS + f];
            for (int ks = 1; ks < nks; ++ks) v += part[ks * L.RP * L.PS + r * L.PS + f];
            v += bias_s[col0 + f];
            if (a.relu) v = fmaxf(v, 0.f);
            part[r * L.PS + f] = v;
            if (a.y && a.y_layout == GPP_NODE_MAJOR) a.y[(row0 + r) * GF_C + col0 + f] = v;
        }
        __syncthreads();
        if (a.y && a.y_layout == GPP_FEATURE_MAJOR) {
            const int per = ncols * N;
            for (int i = threadIdx.x; i < ns * per; i += GF_FWD_THREADS) {
                const int bl = i / per, rem = i - bl * per;
                const int f = rem / N, n = rem - f * N;
                a.y[((size_t)(s0 + bl) * GF_C + col0 + f) * N + n] = part[(bl * N + n) * L.PS + f];
            }
        }
        GF_MARK(4)
        if (a.wa) {
            // logits[n][b][:] = wa . y[b,n,:] + ba   (decentralplanner.py:309-315); one warp
            // per node row, 4 features per lane, butterfly reduction across the warp
            for (int r = warp; r < R; r += GF_FWD_WARPS) {
                float s[NUM_ACT];
#pragma unroll
                for (int c = 0; c < NUM_ACT; ++c) s[c] = 0.f;
                if (lane * 4 < ncols) {
                    const float4 v = ld_smem4(part + r * L.PS + lane * 4);
#pragma unroll
                    for (int c = 0; c < NUM_ACT; ++c) {
                        const float4 w = ld_smem4(wa_s + c * GF_C + col0 + lane * 4);
                        s[c] = v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
                    }
                }
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
                    for (int c = 0; c < NUM_ACT; ++c) s[c] += __shfl_xor_sync(0xffffffffu, s[c], off);
                }
                if (lane < NUM_ACT) {
                    const int bl = r / N, n = r - bl * N;
                    float o = s[0];
#pragma unroll
                    for (int c = 1; c < NUM_ACT; ++c) o = (lane == c) ? s[c] : o;
                    if (a.csplit == 1)
                        a.logits[((size_t)n * a.B + (s0 + bl)) * NUM_ACT + lane] = o + ba_s[lane];
                    else
                        a.lpart[((size_t)half * a.B * N + row0 + r) * NUM_ACT + lane] = o;
                }
            }
            if (a.csplit > 1) {
                __threadfence();
                __syncthreads();
                if (threadIdx.x == 0) {
                    const unsigned int t = atomicAdd(&a.tickets[tile], 1u);
                    s_last = (t == (unsigned int)a.csplit - 1u) ? 1u : 0u;
                    if (s_last) a.tickets[tile] = 0u;          // ready for the next launch
                }
                __syncthreads();
                if (s_last) {
                    __threadfence();
                    for (int i = threadIdx.x; i < R * NUM_ACT; i += GF_FWD_THREADS) {
                        const int r = i / NUM_ACT, c = i - r * NUM_ACT;
                        float o = ba_s[c];
                        for (int hh = 0; hh < a.csplit; ++hh)
                            o += __ldcg(a.lpart + ((size_t)hh * a.B * N + row0 + r) * NUM_ACT + c);
                        const int bl = r / N, n = r - bl * N;
                        a.logits[((size_t)n * a.B + (s0 + bl)) * NUM_ACT + c] = o;
                    }
                }
            }
        }
        __syncthreads();  // part / z / Ss are reused by the next tile
        GF_MARK(5)
    }
#undef GF_MARK
}

// ---------------------------------------------------------------------------------------
// Generic path (any G, F; N*K*G small enough for smem): one CTA per sample, correctness
// first.  z is kept feature-major [K][G][N] exactly like the reference's z tensor.
// ---------------------------------------------------------------------------------------
struct GfGenericArgs {
    const float* x;
    const void* S;
    const float* w;     // [F][K*G] original layout
    const float* bias;
    float* y;
    int B, N, G, F, K;
    int s_is_f64, x_layout, y_layout, relu;
};

__global__ void __launch_bounds__(GF_THREADS) gf_fwd_generic_kernel(const GfGenericArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* z = reinterpret_cast<float*>(smem_raw);   // [K][G][N]
    float* Ss = z + a.K * a.G * a.N;                  // [N][N]
    const int b = blockIdx.x, N = a.N, G = a.G, F = a.F, K = a.K;
    load_gso_plain(Ss, a.S, a.s_is_f64, (size_t)b * N * N, N * N);
    for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
        const int g = i / N, n = i - g * N;
        z[i] = (a.x_layout == GPP_FEATURE_MAJOR) ? a.x[(size_t)b * G * N + i]
                                                 : a.x[((size_t)b * N + n) * G + g];
    }
    __syncthreads();
    for (int k = 1; k < K; ++k) {
        for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
            const int g = i / N, n = i - g * N;
            float acc = 0.f;
            for (int m = 0; m < N; ++m) acc = fmaf(z[((k - 1) * G + g) * N + m], Ss[m * N + n], acc);
            z[(k * G + g) * N + n] = acc;
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < F * N; i += GF_THREADS) {
        const int f = i / N, n = i - f * N;
        float acc = 0.f;
        const float* wr = a.w + (size_t)f * K * G;
        for (int j = 0; j < K * G; ++j) acc = fmaf(wr[j], z[j * N + n], acc);
        if (a.bias) acc += a.bias[f];
        if (a.relu) acc = fmaxf(acc, 0.f);
        if (a.y_layout == GPP_FEATURE_MAJOR)
            a.y[(size_t)b * F * N + i] = acc;
        else
            a.y[((size_t)b * N + n) * F + f] = acc;
    }
}

// wt[(k*G+g)*F + f] = w[(f*K + k)*G + g]
__global__ void transpose_taps_kernel(const float* __restrict__ w, float* __restrict__ wt, int F,
                                      int KG) {
    __shared__ float t[32][33];
    const int j0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int f = f0 + i, j = j0 + threadIdx.x;
        t[i][threadIdx.x] = (f < F && j < KG) ? w[(size_t)f * KG + j] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int j = j0 + i, f = f0 + threadIdx.x;
        if (f < F && j < KG) wt[(size_t)j * F + f] = t[threadIdx.x][i];
    }
}

// ws[(h*KG + j)*64 + c] = wt[j*128 + h*64 + c]: the two column halves of the k-major taps, each contiguous
__global__ void split_taps_kernel(const float* __restrict__ wt, float* __restrict__ ws, int KG) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= KG * GF_C) return;
    const int j = i / GF_C, f = i - j * GF_C;
    ws[((size_t)(f >> 6) * KG + j) * (GF_C / 2) + (f & 63)] = wt[i];
}

// =======================================================================================
// Backward
//   dZ_k[r,g] = sum_f dY[r,f] w[f,k,g]          (tile_contract against w in its own layout)
//   dX        = dZ_0 + S (dZ_1 + S (dZ_2 + ...))   (Horner; z_k = S^T z_{k-1} => dz_{k-1} += S dz_k)
//   dW[f,k,g] = sum_r dY[r,f] z_k[r,g] ,  db[f] = sum_r dY[r,f]
// =======================================================================================
struct GfBwdDataArgs {
    const float* dy;
    const float* y;      // forward output (ReLU mask) or null
    const float* x;      // for the z recomputation written to zbuf (may be null with zbuf)
    const void* S;
    const float* w;      // [128][K*128]
    float* dx;           // null: skip
    float* zbuf;         // [B*N][K*128] node-major z_k (for the dW GEMM), null: skip
    float* dyeff;        // [B*N][128] node-major masked dY (for the dW GEMM), null: skip
    int B, N, K, TS, num_tiles;
    int s_is_f64, x_layout, y_layout, relu;
};

struct GfBwdSmem {
    int RP, ZS, s_floats;
    __host__ __device__ GfBwdSmem(int N, int K, int TS) {
        RP = ((TS * N + 15) / 16) * 16;
        ZS = K * GF_C + 4;
        s_floats = ((TS * N * N + 3) / 4) * 4;
    }
    __host__ __device__ size_t z_off() const { return 0; }
    __host__ __device__ size_t s_off() const { return sizeof(float) * RP * ZS; }
    __host__ __device__ size_t dy_off() const { return s_off() + sizeof(float) * s_floats; }
    __host__ __device__ size_t total() const { return dy_off() + sizeof(float) * RP * GF_PS; }
};

__global__ void __launch_bounds__(GF_THREADS) gf_bwd_data_kernel(const GfBwdDataArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const GfBwdSmem L(a.N, a.K, a.TS);
    float* z = reinterpret_cast<float*>(smem_raw + L.z_off());   // z_k, later dZ_k
    float* Ss = reinterpret_cast<float*>(smem_raw + L.s_off());
    float* dys = reinterpret_cast<float*>(smem_raw + L.dy_off());
    const int N = a.N, K = a.K, ZS = L.ZS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
        const int s0 = tile * a.TS;
        const int ns = min(a.TS, a.B - s0);
        const int R = ns * N;
        const int RP = ((R + 15) >> 4) << 4;
        const size_t row0 = (size_t)s0 * N;

        load_gso_plain(Ss, a.S, a.s_is_f64, (size_t)s0 * N * N, ns * N * N);
        // masked upstream gradient, node-major rows
        if (a.y_layout == GPP_NODE_MAJOR) {
            for (int i = threadIdx.x; i < R * GF_C; i += GF_THREADS) {
                const int r = i >> 7, f = i & 127;
                float v = a.dy[row0 * GF_C + i];
                if (a.relu && !(a.y[row0 * GF_C + i] > 0.f)) v = 0.f;
                dys[r * GF_PS + f] = v;
            }
        } else {
            const size_t base = (size_t)s0 * GF_C * N;
            const int per = GF_C * N;
            for (int i = threadIdx.x; i < ns * per; i += GF_THREADS) {
                const int bl = i / per, rem = i - bl * per;
                const int f = rem / N, n = rem - f * N;
                float v = a.dy[base + i];
                if (a.relu && !(a.y[base + i] > 0.f)) v = 0.f;
                dys[(bl * N + n) * GF_PS + f] = v;
            }
        }
        for (int i = threadIdx.x; i < (RP - R) * GF_C; i += GF_THREADS)
            dys[(R + i / GF_C) * GF_PS + (i % GF_C)] = 0.f;
        if (a.zbuf) {  // recompute z_k and spill it for the weight-gradient GEMM
            if (a.x_layout == GPP_NODE_MAJOR) {
                for (int i = threadIdx.x; i < R * GF_C; i += GF_THREADS)
                    z[(i >> 7) * ZS + (i & 127)] = a.x[row0 * GF_C + i];
            } else {
                const float* xp = a.x + (size_t)s0 * GF_C * N;
                const int per = GF_C * N;
                for (int i = threadIdx.x; i < ns * per; i += GF_THREADS) {
                    const int bl = i / per, rem = i - bl * per;
                    const int g = rem / N, n = rem - g * N;
                    z[(bl * N + n) * ZS + g] = xp[i];
                }
            }
        }
        __syncthreads();
        if (a.dyeff)
            for (int i = threadIdx.x; i < R * GF_C; i += GF_THREADS)
                a.dyeff[row0 * GF_C + i] = dys[(i >> 7) * GF_PS + (i & 127)];
        if (a.zbuf) {
            for (int k = 1; k < K; ++k) {
                for (int r = warp; r < R; r += GF_WARPS) {
                    const int bl = r / N, n = r - bl * N;
                    const float* sp = Ss + bl * N * N + n;
                    const float* zp = z + (bl * N) * ZS + (k - 1) * GF_C + lane * 4;
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                    for (int m = 0; m < N; ++m) {
                        const float s = sp[m * N];
                        const float4 v = ld_smem4(zp + m * ZS);
                        acc.x = fmaf(s, v.x, acc.x);
                        acc.y = fmaf(s, v.y, acc.y);
                        acc.z = fmaf(s, v.z, acc.z);
                        acc.w = fmaf(s, v.w, acc.w);
                    }
                    *reinterpret_cast<float4*>(z + r * ZS + k * GF_C + lane * 4) = acc;
                }
                __syncthreads();
            }
            for (int i = threadIdx.x; i < R * K * (GF_C / 4); i += GF_THREADS) {
                const int r = i / (K * 32), q = i - r * (K * 32);
                *reinterpret_cast<float4*>(a.zbuf + (row0 + r) * (size_t)(K * GF_C) + q * 4) =
                    ld_smem4(z + r * ZS + q * 4);
            }
            __syncthreads();
        }
        if (a.dx) {
            // dZ (all taps) = dY . w   -> overwrites z
            tile_contract<false>(dys, GF_PS, GF_C, a.w, K * GF_C, K * GF_C, z, ZS, 0, RP, 1);
            __syncthreads();
            // Horner: u = dZ_{K-1}; u = dZ_k + S u  (in place in slot k), k = K-2 .. 0
            for (int k = K - 2; k >= 0; --k) {
                for (int r = warp; r < R; r += GF_WARPS) {
                    const int bl = r / N, n = r - bl * N;
                    const float* sp = Ss + bl * N * N + n * N;
                    const float* up = z + (bl * N) * ZS + (k + 1) * GF_C + lane * 4;
                    float4 acc = ld_smem4(z + r * ZS + k * GF_C + lane * 4);
                    for (int m = 0; m < N; ++m) {
                        const float s = sp[m];
                        const float4 v = ld_smem4(up + m * ZS);
                        acc.x = fmaf(s, v.x, acc.x);
                        acc.y = fmaf(s, v.y, acc.y);
                        acc.z = fmaf(s, v.z, acc.z);
                        acc.w = fmaf(s, v.w, acc.w);
                    }
                    *reinterpret_cast<float4*>(z + r * ZS + k * GF_C + lane * 4) = acc;
                }
                __syncthreads();
            }
            if (a.x_layout == GPP_NODE_MAJOR) {
                for (int i = threadIdx.x; i < R * GF_C; i += GF_THREADS)
                    a.dx[row0 * GF_C + i] = z[(i >> 7) * ZS + (i & 127)];
            } else {
                float* dp = a.dx + (size_t)s0 * GF_C * N;
                const int per = GF_C * N;
                for (int i = threadIdx.x; i < ns * per; i += GF_THREADS) {
                    const int bl = i / per, rem = i - bl * per;
                    const int g = rem / N, n = rem - g * N;
                    dp[i] = z[(bl * N + n) * ZS + g];
                }
            }
        }
        __syncthreads();
    }
}

// dW partials: grid (chunks, K). CTA (c, k) accumulates, over its row chunk,
//   P[g][f] = sum_r z_k[r][g] dY[r][f]   as a 128x128 tile, 8x8 per thread,
// and (k == 0) the bias column sums.  Partials are reduced in a fixed order (deterministic).
constexpr int DW_ROWS = 16;
__global__ void __launch_bounds__(GF_THREADS)
gf_bwd_weight_kernel(const float* __restrict__ zbuf, const float* __restrict__ dyeff,
                     float* __restrict__ partial, float* __restrict__ bias_partial, int rows,
                     int K, int rows_per_chunk) {
    __shared__ __align__(16) float zs[DW_ROWS][GF_C];
    __shared__ __align__(16) float ds[DW_ROWS][GF_C];
    const int chunk = blockIdx.x, k = blockIdx.y;
    const int r_begin = chunk * rows_per_chunk;
    const int r_end = min(rows, r_begin + rows_per_chunk);
    const int tg = (threadIdx.x >> 4) * 8;   // g0
    const int tf = (threadIdx.x & 15) * 8;   // f0
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float bsum = 0.f;
    for (int r0 = r_begin; r0 < r_end; r0 += DW_ROWS) {
        const int nr = min(DW_ROWS, r_end - r0);
        for (int i = threadIdx.x; i < DW_ROWS * (GF_C / 4); i += GF_THREADS) {
            const int rr = i >> 5, q = i & 31;
            float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), dv = zv;
            if (rr < nr) {
                zv = *reinterpret_cast<const float4*>(zbuf + (size_t)(r0 + rr) * K * GF_C + k * GF_C + q * 4);
                dv = *reinterpret_cast<const float4*>(dyeff + (size_t)(r0 + rr) * GF_C + q * 4);
            }
            *reinterpret_cast<float4*>(&zs[rr][q * 4]) = zv;
            *reinterpret_cast<float4*>(&ds[rr][q * 4]) = dv;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < DW_ROWS; ++rr) {
            const float4 z0 = ld_smem4(&zs[rr][tg]), z1 = ld_smem4(&zs[rr][tg + 4]);
            const float4 d0 = ld_smem4(&ds[rr][tf]), d1 = ld_smem4(&ds[rr][tf + 4]);
            const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
            const float dd[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(zz[i], dd[j], acc[i][j]);
        }
        if (k == 0 && threadIdx.x < GF_C)
            for (int rr = 0; rr < DW_ROWS; ++rr) bsum += ds[rr][threadIdx.x];
        __syncthreads();
    }
    // partial layout [chunk][f][k][g]  (the module's own [F,1,K,G] layout per chunk)
    float* P = partial + (size_t)chunk * GF_C * K * GF_C;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float* row = P + ((size_t)(tf + j) * K + k) * GF_C + tg;
        *reinterpret_cast<float4*>(row) = make_float4(acc[0][j], acc[1][j], acc[2][j], acc[3][j]);
        *reinterpret_cast<float4*>(row + 4) = make_float4(acc[4][j], acc[5][j], acc[6][j], acc[7][j]);
    }
    if (k == 0 && threadIdx.x < GF_C) bias_partial[chunk * GF_C + threadIdx.x] = bsum;
}

__global__ void reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                       int chunks, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += partial[(size_t)c * n + i];
    out[i] = s;
}

// Generic backward (any G/F): one CTA per sample writes dx; dw/db by a second kernel that
// loops over samples per output element (deterministic, slow, correctness-only).
struct GfBwdGenericArgs {
    const float* dy; const float* y; const float* x; const void* S; const float* w;
    float* dx; float* dw; float* db; float* zbuf; float* dyeff;
    int B, N, G, F, K;
    int s_is_f64, x_layout, y_layout, relu;
};

__global__ void __launch_bounds__(GF_THREADS) gf_bwd_generic_sample_kernel(const GfBwdGenericArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x, N = a.N, G = a.G, F = a.F, K = a.K;
    float* z = reinterpret_cast<float*>(smem_raw);  // [K][G][N]: z_k then dZ_k
    float* Ss = z + K * G * N;                       // [N][N]
    float* dys = Ss + N * N;                         // [F][N]
    load_gso_plain(Ss, a.S, a.s_is_f64, (size_t)b * N * N, N * N);
    for (int i = threadIdx.x; i < F * N; i += GF_THREADS) {
        const int f = i / N, n = i - f * N;
        const size_t gi = (a.y_layout == GPP_FEATURE_MAJOR) ? (size_t)b * F * N + i
                                                            : ((size_t)b * N + n) * F + f;
        float v = a.dy[gi];
        if (a.relu && !(a.y[gi] > 0.f)) v = 0.f;
        dys[i] = v;
        a.dyeff[(size_t)b * F * N + i] = v;   // [B][F][N]
    }
    for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
        const int g = i / N, n = i - g * N;
        z[i] = (a.x_layout == GPP_FEATURE_MAJOR) ? a.x[(size_t)b * G * N + i]
                                                 : a.x[((size_t)b * N + n) * G + g];
    }
    __syncthreads();
    for (int k = 1; k < K; ++k) {
        for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
            const int g = i / N, n = i - g * N;
            float acc = 0.f;
            for (int m = 0; m < N; ++m) acc = fmaf(z[((k - 1) * G + g) * N + m], Ss[m * N + n], acc);
            z[(k * G + g) * N + n] = acc;
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < K * G * N; i += GF_THREADS) a.zbuf[(size_t)b * K * G * N + i] = z[i];
    __syncthreads();
    if (!a.dx) return;
    // dZ[k][g][n] = sum_f w[f][k][g] dy[f][n]
    for (int i = threadIdx.x; i < K * G * N; i += GF_THREADS) {
        const int j = i / N, n = i - j * N;
        float acc = 0.f;
        for (int f = 0; f < F; ++f) acc = fmaf(a.w[(size_t)f * K * G + j], dys[f * N + n], acc);
        z[i] = acc;
    }
    __syncthreads();
    // feature-major Horner: u[g][m] = dZ_k[g][m] + sum_n u_{k+1}[g][n] S[m][n]
    for (int k = K - 2; k >= 0; --k) {
        for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
            const int g = i / N, m = i - g * N;
            float acc = z[(k * G + g) * N + m];
            for (int n = 0; n < N; ++n) acc = fmaf(z[((k + 1) * G + g) * N + n], Ss[m * N + n], acc);
            z[(k * G + g) * N + m] = acc;
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < G * N; i += GF_THREADS) {
        const int g = i / N, n = i - g * N;
        if (a.x_layout == GPP_FEATURE_MAJOR)
            a.dx[(size_t)b * G * N + i] = z[i];
        else
            a.dx[((size_t)b * N + n) * G + g] = z[i];
    }
}

__global__ void gf_bwd_generic_weight_kernel(const GfBwdGenericArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over F*K*G (+F for bias)
    const int KG = a.K * a.G, N = a.N;
    if (i < a.F * KG) {
        if (!a.dw) return;
        const int f = i / KG, j = i - f * KG;
        float acc = 0.f;
        for (int b = 0; b < a.B; ++b) {
            const float* zp = a.zbuf + ((size_t)b * KG + j) * N;
            const float* dp = a.dyeff + ((size_t)b * a.F + f) * N;
            for (int n = 0; n < N; ++n) acc = fmaf(zp[n], dp[n], acc);
        }
        a.dw[i] = acc;
    } else if (i < a.F * KG + a.F) {
        if (!a.db) return;
        const int f = i - a.F * KG;
        float acc = 0.f;
        for (int b = 0; b < a.B; ++b) {
            const float* dp = a.dyeff + ((size_t)b * a.F + f) * N;
            for (int n = 0; n < N; ++n) acc += dp[n];
        }
        a.db[f] = acc;
    }
}

// ---------------------------------------------------------------------------------------
// host-side launchers (internal C++ API, also used by planner.cu)
// ---------------------------------------------------------------------------------------
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int pick_tile_samples(int B, int N) {
    // whole samples per tile: as many as keep >= one tile per SM, capped by the 64-row tile
    const int ts_max = GF_MAX_ROWS / N;
    int ts = B / sm_count();
    if (ts < 1) ts = 1;
    if (ts > ts_max) ts = ts_max;
    return ts;
}

int launch_transpose_taps(const float* w, float* wt, int F, int KG, cudaStream_t st) {
    dim3 grid((KG + 31) / 32, (F + 31) / 32), block(32, 8);
    transpose_taps_kernel<<<grid, block, 0, st>>>(w, wt, F, KG);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

int launch_split_taps(const float* wt, float* ws, int KG, cudaStream_t st) {
    const int n = KG * GF_C;
    split_taps_kernel<<<(n + 255) / 256, 256, 0, st>>>(wt, ws, KG);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

static unsigned long long* g_gf_timing = nullptr;  // GPP_GF_TIMING debug counters

// `lpart` ([2][B*N][5] floats) and `tickets` (>= ceil(B / TS) zeroed counters) are the caller's scratch for the
// column-split launch of small batches; without them (or without the fused action MLP) no scratch is needed.
int launch_gf_forward_fast(const float* x, const void* S, int s_is_f64, const float* wt,
                           const float* bias, float* y, const float* wa, const float* ba,
                           float* logits, int B, int N, int K, int x_layout, int y_layout,
                           int relu, int allow_bulk, float* lpart, unsigned int* tickets, const float* wsplit,
                           int pdl, cudaStream_t st) {
    GfFwdArgs a;
    a.wsplit = wsplit;
    a.pdl = pdl;
    a.x = x; a.S = S; a.wt = wt; a.bias = bias; a.y = y; a.wa = wa; a.ba = ba; a.logits = logits;
    a.B = B; a.N = N; a.K = K;
    a.TS = pick_tile_samples(B, N);
    a.num_tiles = (B + a.TS - 1) / a.TS;
    a.s_is_f64 = s_is_f64; a.x_layout = x_layout; a.y_layout = y_layout; a.relu = relu;
    a.bulk_x = (allow_bulk && x_layout == GPP_NODE_MAJOR && aligned16(x)) ? 1 : 0;
    a.bulk_s = (allow_bulk && !s_is_f64 && aligned16(S) && ((N * N) % 4 == 0)) ? 1 : 0;
    // fewer tiles than SMs: let two CTAs share every tile (column halves)
    a.csplit = (2 * a.num_tiles <= sm_count()) ? 2 : 1;
    if (wa && !(lpart && tickets)) a.csplit = 1;
    a.lpart = lpart;
    a.tickets = tickets;
    a.timing = nullptr;
    if (debug_option(DBG_GF_TIMING)) {
        if (!g_gf_timing) {
            GPP_CUDA_OK(cudaMalloc(&g_gf_timing, 64));
            GPP_CUDA_OK(cudaMemset(g_gf_timing, 0, 64));
        }
        a.timing = g_gf_timing;
    }
    if (a.csplit > 1 && GfFwdSmem(N, K, a.TS, a.csplit, 0).total() > 160 * 1024) a.csplit = 1;
    // one tile per CTA in split launches (2 * num_tiles <= SMs): stage the CTA's half of the taps in smem if it fits
    a.w_smem = (a.csplit == 2 && wsplit && GfFwdSmem(N, K, a.TS, 2, 1).total() <= 220 * 1024) ? 1 : 0;
    const GfFwdSmem L(N, K, a.TS, a.csplit, a.w_smem);
    const size_t smem = L.total();
    static SmemConfig smem_cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(gf_fwd_kernel, smem_cfg, smem));
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gf_fwd_kernel, GF_FWD_THREADS, smem) != cudaSuccess ||
        per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
    }
    const int vtiles = a.num_tiles * a.csplit;
    int grid = vtiles < sm_count() * per_sm ? vtiles : sm_count() * per_sm;
    GPP_CUDA_OK(launch_maybe_pdl(gf_fwd_kernel, grid, GF_FWD_THREADS, smem, st, pdl, a));
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp

namespace gpp {
// tensor-core path (graph_filter_tc.cu)
size_t gf_tc_image_floats(int K);
int gf_tc_tile_samples(int N, int K);
int launch_prep_umma_taps(const float* w, float* img, int K, cudaStream_t st);
int launch_gf_forward_tc(const float* x, const void* S, int s_is_f64, const float* wimg, const float* bias,
                         float* y, const float* wa, const float* ba, float* logits, int B, int N, int K,
                         int relu, int allow_bulk, cudaStream_t st);

// fp16-split wgmma pair kernel (graph_filter_pair.cu)
size_t gf_pair_image_bytes(int K);
bool gf_pair_supported(int N, int K);
int launch_prep_pair_taps(const float* w, void* img, int K, cudaStream_t st);
int launch_gf_forward_pair(const float* x, const void* S, int s_is_f64, const void* wimg, const float* bias, float* y,
                           const float* wa_host, const float* ba_host, float* logits, int B, int N, int K, int relu,
                           cudaStream_t st);

// debug override for the standalone op (gpp_debug_set_option("gf_mode", m)): 0 auto, 1 CUDA-core, 2 wgmma 3xTF32,
// 3 wgmma pair fp16-split
static int standalone_gf_mode() { return debug_option(DBG_GF_MODE); }
}  // namespace gpp

using namespace gpp;

extern "C" size_t gpp_graph_filter_workspace_bytes(int G, int F, int K) {
    // k-major transposed taps (CUDA-core kernel) or split/swizzled chunk images (tensor-core kernel)
    if (G == GF_C && F == GF_C) {
        const size_t tc = sizeof(float) * gf_tc_image_floats(K), pair = gf_pair_image_bytes(K);
        return tc > pair ? tc : pair;
    }
    return 0;
}

static size_t generic_fwd_smem(int N, int G, int K) { return sizeof(float) * ((size_t)K * G * N + N * N); }

extern "C" int gpp_graph_filter_forward(const float* x, const void* S, int s_is_f64, const float* w,
                                        const float* bias, float* y, int B, int N, int G, int F,
                                        int K, int x_layout, int y_layout, int fuse_relu,
                                        void* workspace, void* stream) {
    GPP_REQUIRE(x && S && w && y, GPP_ERR_INVALID, "graph_filter_forward: null pointer");
    GPP_REQUIRE(B >= 0 && N > 0 && G > 0 && F > 0 && K > 0, GPP_ERR_INVALID,
                "graph_filter_forward: bad sizes B=%d N=%d G=%d F=%d K=%d", B, N, G, F, K);
    if (B == 0) return GPP_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (G == GF_C && F == GF_C && N <= GF_MAX_ROWS) {
        GPP_REQUIRE(workspace && aligned16(workspace), GPP_ERR_INVALID,
                    "graph_filter_forward: a 16-byte aligned workspace is required");
        const int mode = standalone_gf_mode();
        const bool node_major = x_layout == GPP_NODE_MAJOR && y_layout == GPP_NODE_MAJOR;
        GPP_REQUIRE(mode != 3 || (node_major && gf_pair_supported(N, K)), GPP_ERR_UNSUPPORTED,
                    "graph_filter_forward: the CTA-pair kernel needs node-major layouts and a supported N / K (N=%d K=%d)", N, K);
        if (node_major && gf_pair_supported(N, K) && (mode == 3 || (mode == 0 && (size_t)B * N >= 4096))) {
            int rc = launch_prep_pair_taps(w, workspace, K, st);
            if (rc) return rc;
            return launch_gf_forward_pair(x, S, s_is_f64, workspace, bias, y, nullptr, nullptr, nullptr, B, N, K, fuse_relu, st);
        }
        if (x_layout == GPP_NODE_MAJOR && y_layout == GPP_NODE_MAJOR && mode != 1 && gf_tc_tile_samples(N, K) > 0 &&
            (mode == 2 || (size_t)B * N >= 4096)) {
            float* img = reinterpret_cast<float*>(workspace);
            int rc = launch_prep_umma_taps(w, img, K, st);
            if (rc) return rc;
            return launch_gf_forward_tc(x, S, s_is_f64, img, bias, y, nullptr, nullptr, nullptr, B, N, K, fuse_relu, 1, st);
        }
        float* wt = reinterpret_cast<float*>(workspace);
        int rc = launch_transpose_taps(w, wt, F, K * G, st);
        if (rc) return rc;
        return launch_gf_forward_fast(x, S, s_is_f64, wt, bias, y, nullptr, nullptr, nullptr, B, N, K,
                                      x_layout, y_layout, fuse_relu, 1, nullptr, nullptr, nullptr, 0, st);
    }
    const size_t smem = generic_fwd_smem(N, G, K);
    GPP_REQUIRE(smem <= 200 * 1024, GPP_ERR_UNSUPPORTED,
                "graph_filter_forward: N*K*G = %d*%d*%d does not fit the generic kernel's shared memory",
                N, K, G);
    GPP_CUDA_OK(cudaFuncSetAttribute(gf_fwd_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    GfGenericArgs a;
    a.x = x; a.S = S; a.w = w; a.bias = bias; a.y = y;
    a.B = B; a.N = N; a.G = G; a.F = F; a.K = K;
    a.s_is_f64 = s_is_f64; a.x_layout = x_layout; a.y_layout = y_layout; a.relu = fuse_relu;
    gf_fwd_generic_kernel<<<B, GF_THREADS, smem, st>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

static int dw_chunks(int rows) {
    int c = (rows + DW_ROWS - 1) / DW_ROWS;
    const int cap = 2 * sm_count() / 3 + 1;
    return c < cap ? (c < 1 ? 1 : c) : cap;
}

extern "C" size_t gpp_graph_filter_backward_workspace_bytes(int B, int N, int G, int F, int K) {
    const size_t rows = (size_t)B * N;
    if (G == GF_C && F == GF_C && N <= GF_MAX_ROWS) {
        const size_t chunks = dw_chunks((int)rows);
        return sizeof(float) * (rows * K * GF_C + rows * GF_C + chunks * GF_C * K * GF_C + chunks * GF_C);
    }
    return sizeof(float) * (rows * K * G + rows * F);
}

extern "C" int gpp_graph_filter_backward(const float* dy, const float* y, const float* x, const void* S,
                                         int s_is_f64, const float* w, float* dx, float* dw,
                                         float* dbias, int B, int N, int G, int F, int K, int x_layout,
                                         int y_layout, int fuse_relu, void* workspace, void* stream) {
    GPP_REQUIRE(dy && x && S && w, GPP_ERR_INVALID, "graph_filter_backward: null pointer");
    GPP_REQUIRE(!fuse_relu || y, GPP_ERR_INVALID, "graph_filter_backward: fuse_relu needs the forward output");
    GPP_REQUIRE(B >= 0 && N > 0 && G > 0 && F > 0 && K > 0, GPP_ERR_INVALID,
                "graph_filter_backward: bad sizes");
    GPP_REQUIRE(workspace, GPP_ERR_INVALID, "graph_filter_backward: workspace required");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (B == 0) {
        if (dw) GPP_CUDA_OK(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)F * K * G, st));
        if (dbias) GPP_CUDA_OK(cudaMemsetAsync(dbias, 0, sizeof(float) * F, st));
        return GPP_OK;
    }
    const size_t rows = (size_t)B * N;
    float* ws = reinterpret_cast<float*>(workspace);
    const bool need_w = dw || dbias;
    if (G == GF_C && F == GF_C && N <= GF_MAX_ROWS) {
        GPP_REQUIRE(aligned16(w) && aligned16(workspace), GPP_ERR_INVALID,
                    "graph_filter_backward: w and workspace must be 16-byte aligned");
        float* zbuf = ws;
        float* dyeff = zbuf + rows * K * GF_C;
        float* partial = dyeff + rows * GF_C;
        const int chunks = dw_chunks((int)rows);
        float* bias_partial = partial + (size_t)chunks * GF_C * K * GF_C;
        GfBwdDataArgs a;
        a.dy = dy; a.y = y; a.x = x; a.S = S; a.w = w; a.dx = dx;
        a.zbuf = need_w ? zbuf : nullptr;
        a.dyeff = need_w ? dyeff : nullptr;
        a.B = B; a.N = N; a.K = K;
        a.TS = pick_tile_samples(B, N);
        a.num_tiles = (B + a.TS - 1) / a.TS;
        a.s_is_f64 = s_is_f64; a.x_layout = x_layout; a.y_layout = y_layout; a.relu = fuse_relu;
        const GfBwdSmem L(N, K, a.TS);
        const size_t smem = L.total();
        static SmemConfig smem_cfg;
        GPP_CUDA_OK(ensure_dynamic_smem(gf_bwd_data_kernel, smem_cfg, smem));
        int per_sm = (int)(220 * 1024 / (smem + 1024));
        if (per_sm < 1) per_sm = 1;
        if (per_sm > 4) per_sm = 4;
        const int grid = a.num_tiles < sm_count() * per_sm ? a.num_tiles : sm_count() * per_sm;
        gf_bwd_data_kernel<<<grid, GF_THREADS, smem, st>>>(a);
        GPP_LAUNCH_CHECK();
        if (need_w) {
            const int rpc = (((int)rows + chunks - 1) / chunks + DW_ROWS - 1) / DW_ROWS * DW_ROWS;
            const int used = ((int)rows + rpc - 1) / rpc;
            gf_bwd_weight_kernel<<<dim3(used, K), GF_THREADS, 0, st>>>(zbuf, dyeff, partial, bias_partial,
                                                                         (int)rows, K, rpc);
            GPP_LAUNCH_CHECK();
            if (dw) {
                const int n = GF_C * K * GF_C;
                reduce_partials_kernel<<<(n + 255) / 256, 256, 0, st>>>(partial, dw, used, n);
                GPP_LAUNCH_CHECK();
            }
            if (dbias) {
                reduce_partials_kernel<<<1, GF_C, 0, st>>>(bias_partial, dbias, used, GF_C);
                GPP_LAUNCH_CHECK();
            }
        }
        return GPP_OK;
    }
    const size_t smem = sizeof(float) * ((size_t)K * G * N + N * N + (size_t)F * N);
    GPP_REQUIRE(smem <= 200 * 1024, GPP_ERR_UNSUPPORTED,
                "graph_filter_backward: sizes do not fit the generic kernel's shared memory");
    GPP_CUDA_OK(cudaFuncSetAttribute(gf_bwd_generic_sample_kernel,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GfBwdGenericArgs a;
    a.dy = dy; a.y = y; a.x = x; a.S = S; a.w = w; a.dx = dx; a.dw = dw; a.db = dbias;
    a.zbuf = ws; a.dyeff = ws + rows * K * G;
    a.B = B; a.N = N; a.G = G; a.F = F; a.K = K;
    a.s_is_f64 = s_is_f64; a.x_layout = x_layout; a.y_layout = y_layout; a.relu = fuse_relu;
    gf_bwd_generic_sample_kernel<<<B, GF_THREADS, smem, st>>>(a);
    GPP_LAUNCH_CHECK();
    if (need_w) {
        const int n = F * K * G + F;
        gf_bwd_generic_weight_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
        GPP_LAUNCH_CHECK();
    }
    return GPP_OK;
}

// debug: per-phase cycle totals of block 0 of gf_fwd_kernel since the last call (only filled when GPP_GF_TIMING is
// set): prologue, x/S staging, propagate, tap contraction, epilogue, action MLP + ticket merge.
extern "C" int gpp_debug_gf_timing(unsigned long long* out6) {
    if (!gpp::g_gf_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out6, gpp::g_gf_timing, 48, cudaMemcpyDeviceToHost);
    cudaMemset(gpp::g_gf_timing, 0, 64);
    return GPP_OK;
}
