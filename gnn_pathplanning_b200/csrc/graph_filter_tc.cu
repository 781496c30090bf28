// Tensor-core (wgmma, Hopper) fused graph filter.
//
// Same contract as gf_fwd_kernel (graph_filter.cu; BatchLSIGF, reference utils/graphUtils/graphML.py:2273-2367,
// + ReLU + the 128->5 action MLP), node-major input, G = F = 128.
//
// Algebra: the graph shift acts on the node index and the taps on the feature index, so they commute:
//     y = sum_k (S^k)^T-shift( x . W_k^T )        instead of        sum_k ( (S^k)^T-shift x ) . W_k^T
// "filter, then propagate".  Per tap the dense part U_k = X[128 rows,128] . W_k^T is one GEMM whose A operand is the
// raw x tile (no per-tap operand to build); the N-term neighbour sums of U_k run afterwards on the CUDA cores.
//
//   * fp32 parity through split precision (3xTF32): operands are split into hi = tf32(v), lo = tf32(v-hi);
//     U += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo, fp32 accumulation in registers (dropped lo.lo term: 2^-22).
//   * B operand (taps): pre-split, pre-swizzled 32 KB chunk images (hi | lo) prepared once per weight update, so a
//     linear copy lands them in the canonical SWIZZLE_128B K-major layout; a 2-stage ring of 16-byte cp.async copies
//     runs one chunk ahead of the MMAs.
//   * A operand: each 128 x 32 chunk of x is read from global memory (coalesced float4), split and stored swizzled
//     into a 2-stage ring.
//   * warp-specialised: 8 producer warps stage operands and arrive on "full" mbarriers; one MMA warpgroup (warps
//     8-11) runs wgmma into a 128 x 128 register accumulator (two M = 64 halves), releases ring stages on "done"
//     mbarriers and, after the 4 chunks of a tap, hands U_k to the producers through shared memory.
//   * epilogue: every producer thread owns one node row x 64 features: U_0 + bias + sum_k sum_m S^k[m,n] U_k[m,:]
//     accumulated tap by tap, ReLU, optional y store, and the in-thread 128->5 action reduction (two half-rows
//     combined through shared memory).
#include "common.cuh"
#include "tc_common.cuh"

#include <stdlib.h>

namespace gpp {

constexpr int TC_THREADS = 256;           // producer / epilogue threads (+ the MMA warpgroup)
constexpr int TC_MMA_THREADS = 128;
constexpr int TC_M = 128;                  // node rows per tile (two wgmma M = 64 halves)
constexpr int TC_C = 128;                  // G = F = 128 (wgmma N per tap)
constexpr int TC_CHUNK_K = 32;             // reduction elements per chunk (128 bytes of tf32)
constexpr int TC_NCC = TC_C / TC_CHUNK_K;  // 4 A chunks per tile
constexpr int TC_OP_BYTES = TC_M * 128;    // one operand half (hi or lo) of one chunk: 16 KB
constexpr int TC_STAGE_BYTES = 2 * TC_OP_BYTES;   // hi | lo
constexpr int TC_NS = 2;                   // ring depth (A and B stages of one item share a slot)
constexpr int TC_RING_BYTES = 2 * TC_NS * TC_STAGE_BYTES;   // 128 KB
constexpr int TC_U_BYTES = TC_M * TC_C * 4;                 // U_k handed to the epilogue: 64 KB
constexpr int TC_MAX_K = 4;
constexpr int TC_ACT = 5;

// ---------------------------------------------------------------------------------------
// B-operand images: img[c] = { hi[128 x 32] , lo[128 x 32] } in SWIZZLE_128B K-major layout; chunk
// c = k*4 + cc holds w[f][k][g] for g in [32cc, 32cc+32)  (w = the module's [F,1,K,G] taps).
// ---------------------------------------------------------------------------------------
__global__ void prep_umma_taps_kernel(const float* __restrict__ w, float* __restrict__ img, int KG) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;     // one (f, kg) element each
    if (idx >= TC_C * KG) return;
    const int f = idx / KG, kg = idx - f * KG;
    const int c = kg / TC_CHUNK_K, kk = kg - c * TC_CHUNK_K;
    float hi, lo;
    split_tf32(w[idx], hi, lo);
    const uint32_t off = sw128_offset(f, kk >> 2) / 4 + (kk & 3);
    float* base = img + (size_t)c * (TC_STAGE_BYTES / 4);
    base[off] = hi;
    base[TC_OP_BYTES / 4 + off] = lo;
}

struct GfTcArgs {
    const float* x;       // [B*N][128] node-major
    const void* S;
    const float* wimg;    // chunk images
    const float* bias;    // [128] or null
    float* y;             // [B*N][128] node-major or null
    const float* wa;      // [5][128] or null
    const float* ba;
    float* logits;        // [N][B][5]
    int B, N, K, TS, num_tiles;
    int s_is_f64, relu;
    unsigned long long* timing;   // optional [8] cycle counters (debug), null in production
};

struct GfTcSmem {
    uint32_t sk_floats;
    __host__ __device__ GfTcSmem(int N, int K, int TS) {
        sk_floats = (uint32_t)(((K > 1 ? (K - 1) : 0) * TS * N * N + 3) / 4 * 4);
    }
    __host__ __device__ uint32_t a_stage(int s) const { return (uint32_t)s * TC_STAGE_BYTES; }
    __host__ __device__ uint32_t b_stage(int s) const { return (uint32_t)(TC_NS + s) * TC_STAGE_BYTES; }
    __host__ __device__ uint32_t u_off() const { return TC_RING_BYTES; }
    __host__ __device__ uint32_t sk_off() const { return u_off() + TC_U_BYTES; }
    __host__ __device__ uint32_t misc_off() const { return sk_off() + sk_floats * 4; }   // bias, wa, ba, plog
    __host__ __device__ uint32_t bar_off() const {
        return misc_off() + (TC_C + TC_ACT * TC_C + 8 + TC_M * TC_ACT) * 4;
    }
    __host__ __device__ uint32_t total() const { return bar_off() + 256 + 1024; }          // + alignment slack
};

// word offset of float4 `f4` of row `row` in a [128][128] fp32 tile whose float4 columns are XOR-swizzled by
// the row (conflict-free for row-per-lane writes and for same-row broadcast reads)
__device__ __forceinline__ int usm_off(int row, int f4) { return row * TC_C + ((f4 ^ (row & 31)) << 2); }

// One arrival per producer WARP (barrier count = 8) and one polling lane per warp: 256 threads arriving on /
// polling the same mbarrier serialise in the shared-memory atomic unit.
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0)
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
    if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
    __syncwarp();
}
__device__ __forceinline__ void producers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void mma_group_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }

// 128 x 128 accumulator of the MMA warpgroup (acc[h] = rows 64 h .. 64 h + 63) -> U tile in shared memory
__device__ __forceinline__ void tc_store_u(float* usm, const float (&acc)[2][64], int t) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int row = 64 * h + wg_row(t, i), col = wg_col(t, i);
            *reinterpret_cast<float2*>(usm + usm_off(row, col >> 2) + (col & 3)) = make_float2(acc[h][i], acc[h][i + 1]);
        }
}

// Warp roles: warps 0-7 (256 threads) = producers (B cp.async, A split/store) and epilogue; warps 8-11 = MMA
// warpgroup.  Item q = (tile, tap k, chunk cc) in that order; its A and B operands share ring slot q % 2.
__global__ void __launch_bounds__(TC_THREADS + TC_MMA_THREADS, 1) gf_fwd_tc_kernel(const GfTcArgs a) {
    extern __shared__ unsigned char smem_raw_tc[];
    const uint32_t raw = smem_u32(smem_raw_tc);
    unsigned char* sm = smem_raw_tc + (((raw + 1023u) & ~1023u) - raw);      // 1024-byte aligned base
    const GfTcSmem L(a.N, a.K, a.TS);
    float* usm = reinterpret_cast<float*>(sm + L.u_off());
    float* sk = reinterpret_cast<float*>(sm + L.sk_off());
    float* bias_s = reinterpret_cast<float*>(sm + L.misc_off());
    float* wa_s = bias_s + TC_C;
    float* ba_s = wa_s + TC_ACT * TC_C;
    float* plog = ba_s + 8;                                    // [128][5] partial logits of the upper half-rows
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + L.bar_off());
    uint64_t* full = bars;                        // [TC_NS] every producer warp stored its A part and saw its B copies land
    uint64_t* done = bars + TC_NS;                // [TC_NS] the MMAs that read the slot have completed
    uint64_t* u_full = bars + 2 * TC_NS;          // U_k of the current tap is in shared memory
    uint64_t* u_free = u_full + 1;                // the epilogue is done with it
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int N = a.N, K = a.K;
    const int nitems = TC_NCC * K;

    if (tid == 0) {
        for (int i = 0; i < TC_NS; ++i) {
            mbar_init(&full[i], TC_THREADS / 32);
            mbar_init(&done[i], 1);
        }
        mbar_init(u_full, 1);
        mbar_init(u_free, 1);
        fence_mbar_init();
    }
    for (int i = tid; i < TC_C; i += blockDim.x) bias_s[i] = a.bias ? a.bias[i] : 0.f;
    if (a.wa) {
        for (int i = tid; i < TC_ACT * TC_C; i += blockDim.x) wa_s[i] = a.wa[i];
        if (tid < TC_ACT) ba_s[tid] = a.ba[tid];
    }
    __syncthreads();

    if (warp >= TC_THREADS / 32) {
        // =============================== MMA warpgroup ===============================
        const int t = tid - TC_THREADS;
        float acc[2][64];
        uint32_t q = 0, nu = 0;
        for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
            for (int it = 0; it < nitems; ++it, ++q) {
                const int cc = it % TC_NCC;
                const int s = q % TC_NS;
                mbar_wait(&full[s], (q / TC_NS) & 1);
                const uint32_t sa = smem_u32(sm + L.a_stage(s)), sb = smem_u32(sm + L.b_stage(s));
                const uint64_t b_hi = gmma_desc_sw128(sb), b_lo = gmma_desc_sw128(sb + TC_OP_BYTES);
                wgmma_fence();
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    // rows 64 h ..: 8 groups of 1024 bytes further; +32 bytes (2 x 16 B units) per K = 8 step
                    const uint64_t a_hi = gmma_desc_sw128(sa + h * 8192), a_lo = gmma_desc_sw128(sa + TC_OP_BYTES + h * 8192);
#pragma unroll
                    for (int ks = 0; ks < TC_CHUNK_K / 8; ++ks)
                        wgmma_tf32<128>(acc[h], a_hi + 2 * ks, b_hi + 2 * ks, (cc | ks) != 0);
#pragma unroll
                    for (int ks = 0; ks < TC_CHUNK_K / 8; ++ks) wgmma_tf32<128>(acc[h], a_lo + 2 * ks, b_hi + 2 * ks, 1u);
#pragma unroll
                    for (int ks = 0; ks < TC_CHUNK_K / 8; ++ks) wgmma_tf32<128>(acc[h], a_hi + 2 * ks, b_lo + 2 * ks, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                mma_group_sync();
                if (t == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&done[s])) : "memory");
                if (cc == TC_NCC - 1) {
                    if (nu >= 1) mbar_wait(u_free, (nu - 1) & 1);
                    tc_store_u(usm, acc, t);
                    mma_group_sync();
                    if (t == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(u_full)) : "memory");
                    ++nu;
                }
            }
        }
    } else {
        // =============================== producers + epilogue ===============================
        uint32_t q = 0;     // items staged so far
        uint32_t nu = 0;    // U tiles consumed
        const int j = tid & 7;      // 16-byte column of this thread inside a 128-byte operand row

        auto issue_b = [&](uint32_t qq, int c) {      // B chunk c of the tap images -> slot of item qq
            const int bs = qq % TC_NS;
            if (qq >= TC_NS) mbar_wait_warp(&done[bs], ((qq / TC_NS) - 1) & 1);
            const char* src = reinterpret_cast<const char*>(a.wimg) + (size_t)c * TC_STAGE_BYTES;
            const uint32_t dst = smem_u32(sm + L.b_stage(bs));
#pragma unroll
            for (int i = 0; i < TC_STAGE_BYTES / (16 * TC_THREADS); ++i) {
                const int u = tid + i * TC_THREADS;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + u * 16), "l"(src + (size_t)u * 16)
                             : "memory");
            }
        };

        unsigned long long tacc[6] = {0, 0, 0, 0, 0, 0};
        for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
            const int s0 = tile * a.TS;
            const int ns = min(a.TS, a.B - s0);
            const int R = ns * N;
            const size_t row0 = (size_t)s0 * N;
            const long long t0 = clock64();
            const int r = (warp & 3) * 32 + lane;        // node row of the tile
            const int h = warp >> 2;                     // which 64-feature half of the row
            float acc[64];
            long long t_wait = 0, t_prop = 0;

            issue_b(q, 0);                                // item (k 0, cc 0): B chunk k * 4 + cc
            asm volatile("cp.async.commit_group;" ::: "memory");
            for (int it = 0; it < nitems; ++it, ++q) {
                const int k = it / TC_NCC, cc = it % TC_NCC;
                if (it + 1 < nitems) issue_b(q + 1, it + 1);   // B runs one item ahead (image chunk index = item index)
                asm volatile("cp.async.commit_group;" ::: "memory");   // (possibly empty) keeps the group count uniform
                const int as = q % TC_NS;
                if (q >= TC_NS) mbar_wait_warp(&done[as], ((q / TC_NS) - 1) & 1);
                unsigned char* stage = sm + L.a_stage(as);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int rr = (tid >> 3) + 32 * i;
                    const float4 xv = (rr < R) ? __ldg(reinterpret_cast<const float4*>(a.x + (row0 + rr) * TC_C +
                                                                                     cc * TC_CHUNK_K + j * 4))
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
                    float4 hi, lo;
                    split_tf32(xv.x, hi.x, lo.x);
                    split_tf32(xv.y, hi.y, lo.y);
                    split_tf32(xv.z, hi.z, lo.z);
                    split_tf32(xv.w, hi.w, lo.w);
                    const uint32_t off = sw128_offset(rr, j);
                    *reinterpret_cast<float4*>(stage + off) = hi;
                    *reinterpret_cast<float4*>(stage + TC_OP_BYTES + off) = lo;
                }
                asm volatile("cp.async.wait_group 1;" ::: "memory");   // this item's B chunk landed
                fence_proxy_async_smem();          // st.shared / cp.async data -> visible to the tensor core
                mbar_arrive(&full[as]);
                if (it == 1 && K > 1) {
                    // GSO tile and its powers: only the epilogue needs them, so they are built here, in the shadow of
                    // the first chunk-MMAs, not in front of them
                    const size_t off = (size_t)s0 * N * N;
                    const int cnt = ns * N * N;
                    if (a.s_is_f64) {
                        const double* Sd = reinterpret_cast<const double*>(a.S) + off;
                        for (int i = tid; i < cnt; i += TC_THREADS) sk[i] = static_cast<float>(Sd[i]);
                    } else {
                        const float* Sf = reinterpret_cast<const float*>(a.S) + off;
                        for (int i = tid; i < cnt; i += TC_THREADS) sk[i] = Sf[i];
                    }
                    for (int p = 1; p < K - 1; ++p) {           // sk[p] = S^(p+1) = S^p . S
                        producers_sync();
                        const float* prev = sk + (size_t)(p - 1) * a.TS * N * N;
                        float* cur = sk + (size_t)p * a.TS * N * N;
                        for (int i = tid; i < cnt; i += TC_THREADS) {
                            const int b = i / (N * N), rem = i - b * N * N;
                            const int rr = rem / N, c = rem - rr * N;
                            float sacc = 0.f;
                            for (int m = 0; m < N; ++m)
                                sacc = fmaf(prev[b * N * N + rr * N + m], sk[b * N * N + m * N + c], sacc);
                            cur[i] = sacc;
                        }
                    }
                    producers_sync();
                }
                if (cc == TC_NCC - 1) {
                    // ---- epilogue part of tap k: acc (+)= U_0 + bias, or sum_m S^k[m, n] U_k[(b, m), :]
                    const long long w0 = clock64();
                    mbar_wait_warp(u_full, nu & 1);
                    ++nu;
                    const long long w1 = clock64();
                    if (k == 0) {
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const float4 u = ld_smem4(usm + usm_off(r, h * 16 + i));
                            acc[4 * i] = u.x + bias_s[h * 64 + 4 * i];
                            acc[4 * i + 1] = u.y + bias_s[h * 64 + 4 * i + 1];
                            acc[4 * i + 2] = u.z + bias_s[h * 64 + 4 * i + 2];
                            acc[4 * i + 3] = u.w + bias_s[h * 64 + 4 * i + 3];
                        }
                    } else if (r < R) {
                        const int b = r / N, n = r - b * N;
                        const float* sp = sk + ((size_t)(k - 1) * a.TS + b) * N * N + n;
                        for (int m = 0; m < N; ++m) {
                            const float sv = sp[m * N];
                            const int row = b * N + m;
#pragma unroll
                            for (int i = 0; i < 16; ++i) {
                                const float4 u = ld_smem4(usm + usm_off(row, h * 16 + i));
                                acc[4 * i] = fmaf(sv, u.x, acc[4 * i]);
                                acc[4 * i + 1] = fmaf(sv, u.y, acc[4 * i + 1]);
                                acc[4 * i + 2] = fmaf(sv, u.z, acc[4 * i + 2]);
                                acc[4 * i + 3] = fmaf(sv, u.w, acc[4 * i + 3]);
                            }
                        }
                    }
                    producers_sync();          // every thread is done with U_k
                    if (tid == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(u_free)) : "memory");
                    t_wait += w1 - w0;
                    t_prop += clock64() - w1;
                }
            }
            const long long t1 = clock64();

            // ---- epilogue: ReLU, y, logits ---------------------------------------------------------------
            {
                if (r < R && a.relu) {
#pragma unroll
                    for (int i = 0; i < 64; ++i) acc[i] = fmaxf(acc[i], 0.f);
                }
                if (r < R) {
                    if (a.y) {
                        float4* yp = reinterpret_cast<float4*>(a.y + (row0 + r) * TC_C + h * 64);
#pragma unroll
                        for (int i = 0; i < 16; ++i)
                            yp[i] = make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
                    }
                }
                if (a.wa) {
                    float s5[TC_ACT];
#pragma unroll
                    for (int qa = 0; qa < TC_ACT; ++qa) {
                        float tt = 0.f;
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const float4 w4 = ld_smem4(wa_s + qa * TC_C + h * 64 + 4 * i);
                            tt = fmaf(acc[4 * i], w4.x, tt);
                            tt = fmaf(acc[4 * i + 1], w4.y, tt);
                            tt = fmaf(acc[4 * i + 2], w4.z, tt);
                            tt = fmaf(acc[4 * i + 3], w4.w, tt);
                        }
                        s5[qa] = tt;
                    }
                    if (h == 1) {
#pragma unroll
                        for (int qa = 0; qa < TC_ACT; ++qa) plog[r * TC_ACT + qa] = s5[qa];
                    }
                    producers_sync();
                    if (h == 0 && r < R) {
                        const int b = r / N, n = r - b * N;
                        float* lp = a.logits + ((size_t)n * a.B + (s0 + b)) * TC_ACT;
#pragma unroll
                        for (int qa = 0; qa < TC_ACT; ++qa) lp[qa] = s5[qa] + plog[r * TC_ACT + qa] + ba_s[qa];
                    }
                }
                producers_sync();      // sk and plog are free for the next tile
                const long long t2 = clock64();
                tacc[0] += (t1 - t0) - t_wait - t_prop; tacc[1] += t_wait; tacc[3] += t_prop; tacc[4] += t2 - t1;
                tacc[5] += 1;
            }
        }
        if (a.timing && tid == 0)
            for (int i = 0; i < 6; ++i) atomicAdd(&a.timing[i], tacc[i]);
    }
}

// ---------------------------------------------------------------------------------------
// Self-test of the wgmma plumbing: D[128][128] = A[128][32] . B[128][32]^T for tf32-exact inputs
// (descriptor encoding, SWIZZLE_128B addressing, accumulator fragment mapping) -- used by tests only.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 1) umma_selftest_kernel(const float* __restrict__ A,
                                                               const float* __restrict__ Bm,
                                                               float* __restrict__ D) {
    extern __shared__ unsigned char smem_raw_st[];
    const uint32_t raw = smem_u32(smem_raw_st);
    unsigned char* sm = smem_raw_st + (((raw + 1023u) & ~1023u) - raw);
    const int tid = threadIdx.x;
    for (int i = tid; i < TC_M * 8; i += 128) {
        const int r = i >> 3, jj = i & 7;
        *reinterpret_cast<float4*>(sm + sw128_offset(r, jj)) = *reinterpret_cast<const float4*>(A + r * 32 + jj * 4);
        *reinterpret_cast<float4*>(sm + TC_OP_BYTES + sw128_offset(r, jj)) =
            *reinterpret_cast<const float4*>(Bm + r * 32 + jj * 4);
    }
    fence_proxy_async_smem();
    __syncthreads();
    float acc[2][64];
    const uint32_t sa = smem_u32(sm);
    const uint64_t db = gmma_desc_sw128(sa + TC_OP_BYTES);
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint64_t da = gmma_desc_sw128(sa + h * 8192);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_tf32<128>(acc[h], da + 2 * ks, db + 2 * ks, ks != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 64; ++i) D[(64 * h + wg_row(tid, i)) * TC_C + wg_col(tid, i)] = acc[h][i];
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
static unsigned long long* g_tc_timing = nullptr;
size_t gf_tc_image_floats(int K) { return (size_t)K * TC_C * TC_C * 2; }

int launch_prep_umma_taps(const float* w, float* img, int K, cudaStream_t st) {
    const int n = TC_C * K * TC_C;
    prep_umma_taps_kernel<<<(n + 255) / 256, 256, 0, st>>>(w, img, K * TC_C);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

// Samples per 128-row tile such that the GSO powers fit next to the operand rings; 0 = does not fit.
int gf_tc_tile_samples(int N, int K) {
    if (N > TC_M || K > TC_MAX_K) return 0;
    int ts = TC_M / N;
    const size_t budget = 227 * 1024;
    while (ts > 0 && GfTcSmem(N, K, ts).total() > budget) --ts;
    return ts;
}

int launch_gf_forward_tc(const float* x, const void* S, int s_is_f64, const float* wimg, const float* bias,
                         float* y, const float* wa, const float* ba, float* logits, int B, int N, int K,
                         int relu, int allow_bulk, cudaStream_t st) {
    (void)allow_bulk;
    GfTcArgs a;
    a.TS = gf_tc_tile_samples(N, K);
    GPP_REQUIRE(a.TS > 0, GPP_ERR_UNSUPPORTED, "gf_forward_tc: N=%d K=%d does not fit the tensor-core tile", N, K);
    GPP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15u) == 0, GPP_ERR_INVALID, "gf_forward_tc: x must be 16-byte aligned");
    a.x = x; a.S = S; a.wimg = wimg; a.bias = bias; a.y = y; a.wa = wa; a.ba = ba; a.logits = logits;
    a.B = B; a.N = N; a.K = K;
    a.num_tiles = (B + a.TS - 1) / a.TS;
    a.s_is_f64 = s_is_f64; a.relu = relu;
    a.timing = nullptr;
    if (debug_option(DBG_TC_TIMING)) {
        static unsigned long long* dbuf = nullptr;
        if (!dbuf) { cudaMalloc(&dbuf, 64); cudaMemset(dbuf, 0, 64); }
        a.timing = dbuf;
        g_tc_timing = dbuf;
    }
    const size_t smem = GfTcSmem(N, K, a.TS).total();
    static SmemConfig smem_cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(gf_fwd_tc_kernel, smem_cfg, smem));
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    gf_fwd_tc_kernel<<<grid, TC_THREADS + TC_MMA_THREADS, smem, st>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp

using namespace gpp;

// debug: per-phase cycle totals of gf_fwd_tc_kernel (only filled when GPP_TC_TIMING is set): item staging
// loop, wait for U_k, (unused), propagation, stores+logits, tiles
extern "C" int gpp_debug_tc_timing(unsigned long long* out6) {
    if (!g_tc_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out6, g_tc_timing, 48, cudaMemcpyDeviceToHost);
    cudaMemset(g_tc_timing, 0, 64);
    return GPP_OK;
}

extern "C" int gpp_debug_umma_selftest(const float* A, const float* B, float* D, void* stream) {
    GPP_REQUIRE(A && B && D, GPP_ERR_INVALID, "umma_selftest: null pointer");
    const size_t smem = 2 * TC_OP_BYTES + 1024;
    GPP_CUDA_OK(cudaFuncSetAttribute(umma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    umma_selftest_kernel<<<1, 128, smem, reinterpret_cast<cudaStream_t>(stream)>>>(A, B, D);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}
