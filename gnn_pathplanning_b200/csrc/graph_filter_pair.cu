// Tensor-core graph filter (Hopper wgmma): propagate on the CUDA cores, contract on the tensor cores.
//
// Same contract as gf_fwd_kernel / gf_fwd_tc_kernel (BatchLSIGF, reference utils/graphUtils/graphML.py:2273-2367,
// + the ReLU of decentralplanner.py:221 and optionally the 128->5 action MLP of :303-315), node-major in / out,
// G = F = 128, K <= 3 taps, small graphs (N nodes known at compile time so the propagation lives in registers).
//
//   * 2-way fp16 split with power-of-two scaling instead of 3xTF32: v * 2^e = hi + lo, both fp16 (11 + 11 significant
//     bits, the same 22 bits 3xTF32 keeps), Y += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo at twice the TF32 rate, half the
//     operand bytes.  fp16 has 5 exponent bits, so the scale is chosen per sample from a bound on |z_k| (max|x| times
//     powers of the largest absolute column sum of S) by scout warps that run one tile ahead, per tensor for the taps;
//     both are undone exactly in the epilogue.  Values more than 2^10 below the per-sample maximum lose relative (not
//     absolute) precision; nothing can overflow.
//   * propagate-then-filter: z_k = x.S^k is formed BEFORE the GEMM by the producer warps, entirely in registers (a
//     lane owns 4 features of all N nodes of one sample), split and stored as A-operand rows; the dense part is ONE
//     accumulating GEMM Y[128, 128] = [z_0 | z_1 | z_2][128, 384] . W[384, 128] per tile, and the epilogue is scale,
//     bias, ReLU and the 5-wide MLP only.
//   * the taps (fp16 hi | lo, 64 KB per tap) stream through a 2-slot ring of bulk copies, one 32-feature chunk of all
//     taps per slot; they stay hot in L2.
//
// Warp roles (640 threads per CTA): 0-11 producers (x -> z_k -> fp16 hi|lo operand rows), 12-15 = the MMA warpgroup
// (wgmma into a 128 x 128 register accumulator, then the epilogue straight from its registers), 16 tap loader, 17-19
// scouts (S and S.S staging, scales, L2 prefetch).
// Operand row layout: 128 bytes = [32 x hi | 32 x lo] fp16 of one (tap, 32-feature chunk), SWIZZLE_128B K-major; the
// three products of a K = 16 step differ only in the descriptors' start offsets (+0 / +64 bytes).
#include "common.cuh"
#include "tc_common.cuh"

#include <cuda_fp16.h>

namespace gpp {

constexpr int GP_THREADS = 640;
constexpr int GP_PROD_WARPS = 12;           // warps 0..11: 2 ring groups x 3 sample quads x 2 item kinds
constexpr int GP_EPI_WARP0 = 12;            // warps 12..15: the MMA + epilogue warpgroup
constexpr int GP_LOAD_WARP = 16;
constexpr int GP_SCOUT_WARP0 = 17;          // warps 17..19
constexpr int GP_SCOUT_WARPS = 3;
constexpr int GP_M = 128;                   // node rows per CTA tile
constexpr int GP_C = 128;                   // G = F
constexpr int GP_NCHUNK = 4;                // 32-feature chunks
constexpr int GP_BUNIT = GP_C * 128;        // one (tap, chunk) B operand: 128 rows, 16 KB
constexpr int GP_MAX_K = 3;
constexpr int GP_ACT = 5;
constexpr int GP_SCALE_RING = 8;            // tiles of per-sample inverse scales kept for the epilogue
constexpr int GP_MAX_TS = 16;              // samples per tile (128 / N, N >= 8)
// registers per thread: 96 at launch (640 threads); the three producer warpgroups hand 32 each to the MMA warpgroup,
// whose 128 x 128 fp32 accumulator alone takes 128
constexpr int GP_PROD_REGS = 64, GP_MMA_REGS = 192;
static_assert(3 * GP_PROD_REGS + GP_MMA_REGS + 96 <= 5 * 96, "register pool of the CTA");
constexpr long long GP_WATCHDOG_CYCLES = 1LL << 31;   // ~1 s: a stuck pipeline traps instead of hanging the GPU

struct GpArgs {
    const float* x;           // [B*N][128] node-major
    const void* S;            // [B][N][N] f32 / f64
    const unsigned char* wimg;   // K*4 operand units (prep_pair_taps_kernel), unit (k, chunk c) at (c * K + k)
    const float* wscale;      // {2^e, 2^-e} of the taps
    const float* bias;        // [128] or null
    float* y;                 // [B*N][128] or null
    float* logits;            // [N][B][5] or null
    int B, K, TS, num_tiles;
    int s_is_f64, relu, has_act;
    int ablate;               // debug ("pair_ablate"): 1 skip the propagations, 2 skip the operand stores, 4 skip the x loads, 8 skip the y stores
    unsigned long long* timing;   // optional [16] per-role cycle totals (debug option "tc_timing"), null in production
    float wa[GP_ACT * GP_C];  // action MLP (kernel-parameter constant bank: FFMA operands, no loads)
    float ba[8];
};

// Row m of a staged GSO (or of S.S) holds the N coefficients of z[n] += S[m][n] x[m] in two blocks, one per half of the
// output nodes: [n = 0 .. NA-1 | pad to 4 | n = NA .. N-1 | pad to 4]  (N = 10: NA = 6 -> 12 floats: a 16-byte + an 8-byte
// load for the first half, one 16-byte load for the second).
__host__ __device__ constexpr int gp_na(int N) { return (N + 2) / 2 <= 4 ? (N < 4 ? N : 4) : (N + 2) / 2; }
__host__ __device__ constexpr int gp_slot_b(int N) { return (gp_na(N) + 3) & ~3; }
__host__ __device__ constexpr int gp_np(int N) { return gp_slot_b(N) + ((N - gp_na(N) + 3) & ~3); }
__host__ __device__ constexpr int gp_slot(int N, int n) { return n < gp_na(N) ? n : gp_slot_b(N) + (n - gp_na(N)); }

struct GpSmem {
    uint32_t b_off, a_off, a_unit, s_off, s_bytes, misc_off, bar_off, total;
    __host__ __device__ GpSmem(int N, int K, int TS) {
        b_off = 0;                                          // 2 ring slots of K tap units
        a_off = b_off + 2u * K * GP_BUNIT;
        // an A operand unit keeps only the 8-row groups that hold tile rows (15 of 16 at N = 10): the MMA still reads
        // 128 rows, i.e. up to 1 KB past the unit -- the next unit or the S buffers, always inside this allocation --
        // and what it computes from them lands in accumulator rows nobody reads
        a_unit = (uint32_t)((TS * N + 7) / 8) * 1024u;
        s_off = a_off + 2u * K * a_unit;
        s_bytes = (uint32_t)TS * N * gp_np(N) * 4 * (K > 2 ? 2 : 1);   // per buffer: S, then S.S (third tap)
        misc_off = (s_off + 2 * s_bytes + 15u) & ~15u;      // bias[128] | scale_p[2][TS] | scale_e[8][TS]
        bar_off = misc_off + (GP_C + 2 * GP_MAX_TS + GP_SCALE_RING * GP_MAX_TS) * 4;
        total = bar_off + 512;
    }
};

// ---- mbarrier waits with a watchdog -------------------------------------------------------------------------
// try_wait with a suspend-time hint: the waiting thread sleeps in hardware until the phase completes (or the hint
// elapses) instead of polling, so waiting warps do not take issue slots from the working ones.
constexpr uint32_t GP_SUSPEND_HINT_NS = 1000000;
__device__ __forceinline__ bool gp_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(GP_SUSPEND_HINT_NS)
        : "memory");
    return ok != 0;
}
// Watchdog: a barrier that does not complete within ~1 s traps instead of hanging the GPU.  No printf: a function call
// anywhere in the kernel makes ptxas serialise its wgmma pipelines.  (`id` names the barrier at the call site.)
__device__ __forceinline__ void gp_wait(uint64_t* bar, uint32_t parity, int id) {
    (void)id;
    if (gp_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!gp_try_wait(bar, parity))
        if (clock64() - t0 > GP_WATCHDOG_CYCLES) __trap();
}
__device__ __forceinline__ void gp_wait_warp(uint64_t* bar, uint32_t parity, int id) {
    if ((threadIdx.x & 31) == 0) gp_wait(bar, parity, id);
    __syncwarp();
}
__device__ __forceinline__ void gp_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// fp32 -> fp16 (hi, lo): hi = fp16(v), lo = fp16(v - hi)
__device__ __forceinline__ void gp_split4(const float4 v, uint2& hi, uint2& lo) {
    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    float r0, r1, r2, r3;
    fsub2(v.x, v.y, f01.x, f01.y, r0, r1);
    fsub2(v.z, v.w, f23.x, f23.y, r2, r3);
    const __half2 l01 = __floats2half2_rn(r0, r1), l23 = __floats2half2_rn(r2, r3);
    hi.x = *reinterpret_cast<const uint32_t*>(&h01);
    hi.y = *reinterpret_cast<const uint32_t*>(&h23);
    lo.x = *reinterpret_cast<const uint32_t*>(&l01);
    lo.y = *reinterpret_cast<const uint32_t*>(&l23);
}

// out[i] = sum_m M[m][N0 + i] * in[m] for the CNT output nodes starting at N0 (z = x . M with M = S or S.S,
// graphML.py:2350; 4 features per lane).  SLOT0 = position of coefficient N0 inside a staged row.
template <int N, int N0, int CNT, int SLOT0>
__device__ __forceinline__ void gp_propagate_half(const float* __restrict__ Ms, const float4 (&in)[N], float4 (&out)[CNT]) {
    constexpr int NP = gp_np(N);
#pragma unroll
    for (int m = 0; m < N; ++m) {
        float sv[(CNT + 3) & ~3];
#pragma unroll
        for (int q = 0; q < (CNT + 3) / 4; ++q) {
            if (CNT - 4 * q >= 3) {
                const float4 s4 = ld_smem4(Ms + m * NP + SLOT0 + 4 * q);
                sv[4 * q] = s4.x; sv[4 * q + 1] = s4.y; sv[4 * q + 2] = s4.z; sv[4 * q + 3] = s4.w;
            } else {
                const float2 s2 = *reinterpret_cast<const float2*>(Ms + m * NP + SLOT0 + 4 * q);
                sv[4 * q] = s2.x; sv[4 * q + 1] = s2.y;
            }
        }
#pragma unroll
        for (int i = 0; i < CNT; ++i) {
            if (m == 0) {        // first term: no accumulator to clear
                fmul2_s(sv[i], in[m].x, in[m].y, out[i].x, out[i].y);
                fmul2_s(sv[i], in[m].z, in[m].w, out[i].z, out[i].w);
            } else {
                ffma2_s(sv[i], in[m].x, in[m].y, out[i].x, out[i].y);
                ffma2_s(sv[i], in[m].z, in[m].w, out[i].z, out[i].w);
            }
        }
    }
}
template <int N>
__device__ __forceinline__ void gp_row_addrs(uint32_t unit0, int row0, int l8, uint32_t (&ahi)[N]) {
#pragma unroll
    for (int n = 0; n < N; ++n) ahi[n] = unit0 + sw128_offset(row0 + n, l8 >> 1) + (uint32_t)(l8 & 1) * 8;
}
__device__ __forceinline__ void gp_sts64(uint32_t addr, uint2 v) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}
template <int N>
__device__ __forceinline__ void gp_store_row(const uint32_t (&ahi)[N], int n, uint32_t tap_off, const float4 v) {
    uint2 hi, lo;
    gp_split4(v, hi, lo);
    const uint32_t addr = ahi[n] + tap_off;
    gp_sts64(addr, hi);
    gp_sts64(addr ^ 64u, lo);             // units are 1024-byte aligned: the xor never carries
}
// rows N0 .. N0+CNT-1 of the item's sample: split and store this lane's 4 features
template <int N, int N0, int CNT>
__device__ __forceinline__ void gp_store_rows(const uint32_t (&ahi)[N], uint32_t tap_off, const float4 (&v)[CNT]) {
#pragma unroll
    for (int i = 0; i < CNT; ++i) {
        uint2 hi, lo;
        gp_split4(v[i], hi, lo);
        const uint32_t addr = ahi[N0 + i] + tap_off;
        gp_sts64(addr, hi);
        gp_sts64(addr ^ 64u, lo);         // units are 1024-byte aligned: the xor never carries
    }
}

template <int N, bool TIMING>
__global__ void __launch_bounds__(GP_THREADS, 1) gf_fwd_pair_kernel(const __grid_constant__ GpArgs a) {
    constexpr int NP = gp_np(N);
    extern __shared__ __align__(1024) unsigned char gp_smem_raw[];
    unsigned char* sm = gp_smem_raw;
    if (threadIdx.x == 0 && (smem_u32(sm) & 1023u) != 0) {
        printf("gf_fwd_pair_kernel: dynamic shared memory is not 1024-byte aligned\n");
        __trap();
    }
    constexpr int TS = GP_M / N;          // samples per 128-row tile
    const int K = a.K;
    const GpSmem L(N, K, TS);
    float* bias_s = reinterpret_cast<float*>(sm + L.misc_off);
    float* scale_p = bias_s + GP_C;                       // [2][GP_MAX_TS]  2^e per sample (producers)
    float* scale_e = scale_p + 2 * GP_MAX_TS;             // [GP_SCALE_RING][GP_MAX_TS]  2^-e (epilogue)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + L.bar_off);
    // Ring barriers are per group slot.  Only the warps that have an item in a group touch its barriers (3 at N = 10),
    // so a warp never waits on groups it has no work in.  a_free has FOUR instances per slot, used round-robin by
    // (group >> 1) & 3: a warp that only visits every fourth group cannot tell "phase n-1 still running" from "phase n
    // complete" with a parity wait on a barrier that completes every other group; with an instance that is reused only
    // every 8 groups the ambiguity cannot arise.
    uint64_t* a_full = bars;          // [2] the group's item warps stored all taps of their rows
    uint64_t* a_free = bars + 2;      // [4][2] the MMAs that read the group have completed
    uint64_t* b_full = bars + 10;     // [2] the tap units of the group's chunk have landed
    uint64_t* b_free = bars + 12;     // [2] the MMAs that read them have completed
    uint64_t* s_full = bars + 14;     // [2] the 3 scout warps staged S (+ S.S) + scales of the tile
    uint64_t* s_free = bars + 16;     // [2] 12 producer warps are done with the S buffer
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long t_kernel0 = TIMING ? clock64() : 0;
    unsigned long long tm[4] = {0, 0, 0, 0};          // per-role cycle totals (lane 0 of one warp per role)
#define GP_T0() const long long _t0 = TIMING ? clock64() : 0
#define GP_ACC(i) if (TIMING) tm[i] += (unsigned long long)(clock64() - _t0)
    constexpr int nquad = (TS + 3) >> 2;           // sample quads per tile
    constexpr int ipg = 2 * nquad;                 // items (producer warps) per group: (quad, kind)

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) {
            mbar_init(&a_full[i], ipg);
            for (int q4 = 0; q4 < 4; ++q4) mbar_init(&a_free[q4 * 2 + i], 1);
            mbar_init(&b_full[i], 1);
            mbar_init(&b_free[i], 1);
            mbar_init(&s_full[i], GP_SCOUT_WARPS);
            mbar_init(&s_free[i], GP_PROD_WARPS);
        }
        fence_mbar_init();
    }
    for (int i = tid; i < GP_C; i += GP_THREADS) bias_s[i] = a.bias ? a.bias[i] : 0.f;
    __syncthreads();

    if (warp >= GP_LOAD_WARP) {
      if (warp == GP_LOAD_WARP) {
        // =========================== tap loader: chunk c of every tap per ring slot ===========================
        if (lane == 0) {
            const uint32_t gbytes = (uint32_t)K * GP_BUNIT;
            uint32_t g = 0;
            for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
                for (int c = 0; c < GP_NCHUNK; ++c, ++g) {
                    const int slot = g & 1;
                    if (g >= 2) gp_wait(&b_free[slot], ((g >> 1) - 1) & 1, 12 + slot);
                    mbar_arrive_expect_tx(&b_full[slot], gbytes);
                    bulk_g2s(sm + L.b_off + slot * gbytes, a.wimg + (size_t)c * gbytes, gbytes, &b_full[slot]);
                }
            }
        }
        __syncwarp();
      } else {
        // =========================== scouts: S staging + per-sample scales, one tile ahead ===========================
        // Three warps, each owning every third sample of the tile; their loads hit L2 thanks to the bulk prefetch
        // issued two tiles earlier.
        const int sw = warp - GP_SCOUT_WARP0;
        for (int i = sw * 32 + lane; i < 2 * (int)(L.s_bytes / 4); i += GP_SCOUT_WARPS * 32)
            reinterpret_cast<float*>(sm + L.s_off)[i] = 0.f;        // pad slots of the staged rows: never written again
        asm volatile("bar.sync 1, %0;" ::"r"(GP_SCOUT_WARPS * 32) : "memory");
        int t = 0;
        for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x, ++t) {
            const int s0 = tile * TS;
            const int ns = max(0, min(TS, a.B - s0));
            const int sb = t & 1;
            if (t >= 2) {
                GP_T0();
                gp_wait_warp(&s_free[sb], ((t >> 1) - 1) & 1, 10 + sb);
                GP_ACC(0);
            }
            const long long t_work0 = TIMING ? clock64() : 0;
            if (sw == 0 && lane == 0) {
                // pull the x rows and GSOs of the tile after next into L2: this role's own loads then wait for L2, not for
                // HBM
                const int tile2 = tile + 2 * gridDim.x;
                const long long first = (long long)tile2 * TS;
                if (first < a.B) {
                    const long long cnt = min((long long)TS, (long long)a.B - first);
                    const uint32_t xb = (uint32_t)(cnt * N * GP_C * 4);
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a.x + first * N * GP_C), "r"(xb) : "memory");
                    const size_t ssz = a.s_is_f64 ? 8 : 4;
                    const uint32_t sbytes = (uint32_t)((cnt * N * N * ssz) & ~(size_t)15);
                    const char* sp = reinterpret_cast<const char*>(a.S) + (size_t)first * N * N * ssz;
                    if (sbytes && (reinterpret_cast<uintptr_t>(sp) & 15u) == 0)
                        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(sp), "r"(sbytes) : "memory");
                }
            }
            float* Sd = reinterpret_cast<float*>(sm + L.s_off + sb * L.s_bytes);
            // Software pipeline over this warp's samples: the loads of sample k+1 are issued as soon as the registers of
            // sample k are free (after its |x| fold and the S store), so their latency overlaps the column sums, the
            // scale and the S.S product of sample k.
            float4 xv[N];
            float se[4];
            auto issue_loads = [&](int sl) {
                const bool v = sl < ns;
                const float* xp = a.x + ((size_t)(s0 + sl) * N) * GP_C + lane * 4;
#pragma unroll
                for (int n = 0; n < N; ++n)
                    xv[n] = v ? __ldg(reinterpret_cast<const float4*>(xp + (size_t)n * GP_C)) : make_float4(0.f, 0.f, 0.f, 0.f);
                const size_t so = (size_t)(s0 + sl) * N * N;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int e = 4 * lane + i;
                    const bool ve = v && e < N * N;
                    se[i] = !ve ? 0.f
                                : (a.s_is_f64 ? static_cast<float>(reinterpret_cast<const double*>(a.S)[so + e])   // S.float(), graphML.py:2350
                                              : reinterpret_cast<const float*>(a.S)[so + e]);
                }
            };
            if (sw < TS) issue_loads(sw);
            for (int sl = sw; sl < TS; sl += GP_SCOUT_WARPS) {
                const bool v = sl < ns;
                float mx = 0.f;
                if (v) {
                    // largest |x| of the sample
#pragma unroll
                    for (int n = 0; n < N; ++n) {
                        const float4 q4 = xv[n];
                        mx = fmaxf(mx, fmaxf(fmaxf(fabsf(q4.x), fabsf(q4.y)), fmaxf(fabsf(q4.z), fabsf(q4.w))));
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int e = 4 * lane + i;
                        if (e < N * N) Sd[(sl * N + e / N) * NP + gp_slot(N, e % N)] = se[i];
                    }
                }
                if (sl + GP_SCOUT_WARPS < TS) issue_loads(sl + GP_SCOUT_WARPS);
                __syncwarp();
                float e2 = 1.f, e2inv = 1.f;
                if (v) {
                    // largest absolute column sum of S: |z_k[n]| <= max|z_{k-1}| * sum_m |S[m][n]|
                    float cs = 0.f;
                    if (lane < N) {
#pragma unroll
                        for (int m = 0; m < N; ++m) cs += fabsf(Sd[(sl * N + m) * NP + gp_slot(N, lane)]);
                    }
                    // both are >= 0: the order of the bit patterns is the order of the values (one REDUX each)
                    mx = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(mx)));
                    cs = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(cs)));
                    float bound = mx;
                    const float cm = fmaxf(cs, 1.f);
                    for (int k = 1; k < K; ++k) bound *= cm;
                    // bound in [2^q, 2^(q+1)): scale by 2^(14-q) so that every |z_k| * scale < 2^15 (fp16 max 65504)
                    const uint32_t bits = __float_as_uint(bound);
                    const int q = (int)((bits >> 23) & 0xFF) - 127;
                    if (bound > 0.f && q < 128) {
                        int e = 14 - q;
                        e = max(-100, min(100, e));
                        e2 = __uint_as_float((uint32_t)(e + 127) << 23);
                        e2inv = __uint_as_float((uint32_t)(127 - e) << 23);
                    }
                }
                if (lane == 0) {
                    scale_p[sb * GP_MAX_TS + sl] = e2;
                    scale_e[(t & (GP_SCALE_RING - 1)) * GP_MAX_TS + sl] = e2inv;
                }
                if (K > 2 && v) {
                    // S.S for the third tap: z_2 = (x.S).S = x.(S.S), so the producers form every tap straight from x
                    // lane = (row m, 4-slot part of the staged row): 1 scalar + 1 vector load and 4 FMAs per term
                    float* S2d = Sd + TS * N * NP;
                    constexpr int PARTS = NP / 4;
                    static_assert(N * PARTS <= 32, "one lane per (row, 4-slot part)");
                    if (lane < N * PARTS) {
                        const int m = lane / PARTS, part = lane - m * PARTS;
                        const float* rowm = Sd + (sl * N + m) * NP;
                        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                        for (int jj = 0; jj < N; ++jj) {
                            const float sj = rowm[gp_slot(N, jj)];
                            const float4 r4 = ld_smem4(Sd + (sl * N + jj) * NP + 4 * part);
                            ffma2_s(sj, r4.x, r4.y, acc.x, acc.y);
                            ffma2_s(sj, r4.z, r4.w, acc.z, acc.w);
                        }
                        // carries the sample's scale: tap-2 items use x as it is (unused pad slots stay finite: S pads are zero)
                        fmul2_s(e2, acc.x, acc.y, acc.x, acc.y);
                        fmul2_s(e2, acc.z, acc.w, acc.z, acc.w);
                        *reinterpret_cast<float4*>(S2d + (sl * N + m) * NP + 4 * part) = acc;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) gp_arrive(&s_full[sb]);
            if (TIMING) tm[1] += (unsigned long long)(clock64() - t_work0);
        }
        if (TIMING && a.timing && lane == 0 && sw == 0) { atomicAdd(&a.timing[9], tm[0]); atomicAdd(&a.timing[10], tm[1]); }
      }
    } else if (warp >= GP_EPI_WARP0) {
        // =========================== MMA warpgroup: wgmma -> scale, bias, ReLU -> y / logits ===========================
        // accumulator acc[mh] = rows 64 mh .. 64 mh + 63 of the tile; element i of thread t is (row 64 mh + wg_row(t, i),
        // column wg_col(t, i)); the 4 lanes of a quad hold the 128 columns of the same two rows
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GP_MMA_REGS));
        const int t_wg = tid - 32 * GP_EPI_WARP0;
        const float inv_w = a.wscale[1];
        uint32_t g = 0;
        int t = 0;
        float acc[2][64];
        const long long t_loop0 = TIMING ? clock64() : 0;
        for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x, ++t) {
            const int s0 = tile * TS;
            const int ns = max(0, min(TS, a.B - s0));
            const int R = ns * N;
            for (int c = 0; c < GP_NCHUNK; ++c, ++g) {
                const int slot = g & 1;
                {
                    GP_T0();
                    gp_wait(&a_full[slot], (g >> 1) & 1, slot);
                    gp_wait(&b_full[slot], (g >> 1) & 1, 14 + slot);
                    GP_ACC(0);
                }
                wgmma_fence();
                for (int k = 0; k < K; ++k) {
                    const uint32_t sa = smem_u32(sm + L.a_off + (slot * K + k) * L.a_unit);
                    const uint64_t db = gmma_desc_sw128(smem_u32(sm + L.b_off + (slot * K + k) * GP_BUNIT));
#pragma unroll
                    for (int mh = 0; mh < 2; ++mh) {
                        // descriptor start offsets in 16-byte units: +2 per K = 16 step, +4 = the lo half of the row
                        const uint64_t da = gmma_desc_sw128(sa + mh * 8192);
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) wgmma_f16<128>(acc[mh], da + 2 * ks, db + 2 * ks, (c | k | ks) != 0);
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) wgmma_f16<128>(acc[mh], da + 4 + 2 * ks, db + 2 * ks, 1u);
#pragma unroll
                        for (int ks = 0; ks < 2; ++ks) wgmma_f16<128>(acc[mh], da + 2 * ks, db + 4 + 2 * ks, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                asm volatile("bar.sync 2, 128;" ::: "memory");      // all four warps' MMAs have completed
                if (t_wg == 0) {
                    gp_arrive(&a_free[((g >> 1) & 3) * 2 + slot]);
                    gp_arrive(&b_free[slot]);
                }
            }
            const long long t_work0 = TIMING ? clock64() : 0;
            const size_t row0 = (size_t)s0 * N;
            const bool do_store = a.y != nullptr && !(a.ablate & 8);
            const float* scl = scale_e + (t & (GP_SCALE_RING - 1)) * GP_MAX_TS;
            float acc5[2][2][GP_ACT];
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = 64 * mh + wg_row(t_wg, 2 * hr);
                    const bool valid = r < R;
                    const float sc = scl[valid ? r / N : 0] * inv_w;
                    float p5[GP_ACT] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int i = 4 * jj + 2 * hr, col = wg_col(t_wg, i);
                        float v0 = fmaf(acc[mh][i], sc, bias_s[col]), v1 = fmaf(acc[mh][i + 1], sc, bias_s[col + 1]);
                        if (a.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                        if (a.has_act) {
#pragma unroll
                            for (int o = 0; o < GP_ACT; ++o)
                                p5[o] = fmaf(v1, a.wa[o * GP_C + col + 1], fmaf(v0, a.wa[o * GP_C + col], p5[o]));
                        }
                        if (do_store && valid)
                            *reinterpret_cast<float2*>(a.y + (row0 + r) * GP_C + col) = make_float2(v0, v1);
                    }
#pragma unroll
                    for (int o = 0; o < GP_ACT; ++o) acc5[mh][hr][o] = p5[o];
                }
            if (a.has_act) {
#pragma unroll
                for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                    for (int hr = 0; hr < 2; ++hr) {
                        const int r = 64 * mh + wg_row(t_wg, 2 * hr);
#pragma unroll
                        for (int o = 0; o < GP_ACT; ++o) {
                            float v = acc5[mh][hr][o];
                            v += __shfl_xor_sync(0xffffffffu, v, 1);
                            v += __shfl_xor_sync(0xffffffffu, v, 2);
                            acc5[mh][hr][o] = v;
                        }
                        if ((lane & 3) == 0 && r < R) {
                            const int bl = r / N, n = r - bl * N;
                            float* lp = a.logits + ((size_t)n * a.B + (s0 + bl)) * GP_ACT;
#pragma unroll
                            for (int o = 0; o < GP_ACT; ++o) lp[o] = acc5[mh][hr][o] + a.ba[o];
                        }
                    }
            }
            if (TIMING) tm[1] += (unsigned long long)(clock64() - t_work0);
        }
        if (TIMING) tm[2] = (unsigned long long)(clock64() - t_loop0);
        if (TIMING && a.timing && t_wg == 0) {
            atomicAdd(&a.timing[4], tm[0]); atomicAdd(&a.timing[6], tm[2]); atomicAdd(&a.timing[8], tm[1]);
            atomicAdd(&a.timing[11], (unsigned long long)t);
        }
    } else {
        // =========================== producers: x -> z_k -> fp16 hi|lo operand rows ===========================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GP_PROD_REGS));
        // An item = 4 samples x one 32-feature chunk of one tile: lane (ql, l8) owns features 4*l8 .. 4*l8+3 of all N
        // nodes of sample ql.  Every tap is formed straight from x (z_1 = x.S, z_2 = x.(S.S)), one half of the output
        // nodes at a time, so the live state is x (N x 4) + half a tap ((N+2)/2 x 4) + N row addresses.
        constexpr int NA = gp_na(N), NB = N - NA, SLOT_B = gp_slot_b(N);
        constexpr int ipt = ipg * GP_NCHUNK;           // items per tile
        static_assert(2 * ipg == GP_PROD_WARPS, "producer warps = the items of the two ring groups");
        static_assert((TS % 4) == 0, "item = 4 whole samples");
        // An item = (tile, 32-feature chunk, quad of 4 samples, kind): kind 0 stores the first half of the rows of tap 0
        // (x) and tap 1 (x.S), kind 1 the other rows of tap 0 and tap 2 (x.(S.S)) -- every tap comes straight from x, so the
        // two kinds are independent and run on two warps (what bounds the ring is the LATENCY of an item: a slot is busy from the first operand store until the
        // MMAs that read it have completed).  Warp w always works on ring slot w / 6, quad (w % 6) % 3, kind (w % 6) / 3;
        // its items are I = w, w + 12, ... of the CTA's sequence (tile I / 24, chunk (I % 24) / 6).
        // lanes 0-7 | 8-15 | 16-23 | 24-31 work for samples 0 | 2 | 1 | 3 of the quad: a 64-bit shared store is served one
        // half-warp at a time, and rows 2 samples (20 rows) apart differ in bit 2 of (row & 7), i.e. land in opposite
        // 64-byte halves of the 128-byte swizzled row -- every operand store is then conflict-free
        const int ql = ((lane >> 3) & 1) * 2 + (lane >> 4);
        const int l8 = lane & 7;
        const int slot = warp / ipg;
        const int kind = (warp % ipg) / nquad;
        const int sl = ((warp % ipg) % nquad) * 4 + ql;     // sample of the tile this lane works for, in every item
        int ntile_seq = 0;
        for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) ++ntile_seq;
        const int total_items = ntile_seq * ipt;
        uint32_t ahi0[N];                              // operand row addresses of tap 0 (same rows, same slot every item)
        gp_row_addrs<N>(smem_u32(sm + L.a_off + (size_t)slot * K * L.a_unit), sl * N, l8, ahi0);
        const bool has_work = kind == 0 || K > 2;      // (K < 3: the kind-1 warps only store their half of tap 0)
        const bool st_ok = !(a.ablate & 2);
        int cur_tile = -1;
        for (int I = warp; I < total_items; I += GP_PROD_WARPS) {
            const long long t_item0 = TIMING ? clock64() : 0;
            const int tt = I / ipt, c = (I - tt * ipt) / ipg;
            const uint32_t g = (uint32_t)(tt * GP_NCHUNK + c);
            const int sb = tt & 1;
            const int smp = (blockIdx.x + tt * (int)gridDim.x) * TS + sl;
            const bool sv = smp < a.B && !(a.ablate & 4);
            float4 xv[N];
            const float* xp = a.x + ((size_t)smp * N) * GP_C + c * 32 + l8 * 4;
#pragma unroll
            for (int n = 0; n < N; ++n)
                xv[n] = sv ? __ldg(reinterpret_cast<const float4*>(xp + (size_t)n * GP_C)) : make_float4(0.f, 0.f, 0.f, 0.f);
            if (tt != cur_tile) {
                if (cur_tile >= 0) {                   // done with the S buffer of the previous tile
                    __syncwarp();
                    if (lane == 0) gp_arrive(&s_free[cur_tile & 1]);
                }
                GP_T0();
                gp_wait_warp(&s_full[sb], (tt >> 1) & 1, 8 + sb);
                GP_ACC(0);
                cur_tile = tt;
            }
            // Tap 0 (the scaled x itself) is split between the two kinds -- kind 0: rows [0, H0) + tap 1, kind 1: rows
            // [H0, N) + tap 2 -- so that both warps of an item carry the same number of instructions (an item's LATENCY is
            // what the ring waits for).  Tap 1 needs the scaled x; the staged S.S already carries the scale.
            constexpr int H0 = N / 2;
            const float scale = sv ? scale_p[sb * GP_MAX_TS + sl] : 1.f;
            if (kind == 0) {
#pragma unroll
                for (int n = 0; n < N; ++n) {
                    fmul2_s(scale, xv[n].x, xv[n].y, xv[n].x, xv[n].y);
                    fmul2_s(scale, xv[n].z, xv[n].w, xv[n].z, xv[n].w);
                }
            }
            const float* Ms = reinterpret_cast<const float*>(sm + L.s_off + sb * L.s_bytes) + (size_t)sl * N * NP;
            if (g >= 2) {       // the MMAs of group g - 2 (same ring slot) must have completed
                GP_T0();
                gp_wait_warp(&a_free[(((g - 2) >> 1) & 3) * 2 + slot], ((g - 2) >> 3) & 1, 2 + slot);
                GP_ACC(1);
            }
            if (kind == 0) {
#pragma unroll
                for (int n = 0; n < H0; ++n) {
                    if (st_ok) gp_store_row<N>(ahi0, n, 0u, xv[n]);
                }
            } else {
#pragma unroll
                for (int n = H0; n < N; ++n) {
                    float4 t;
                    fmul2_s(scale, xv[n].x, xv[n].y, t.x, t.y);
                    fmul2_s(scale, xv[n].z, xv[n].w, t.z, t.w);
                    if (st_ok) gp_store_row<N>(ahi0, n, 0u, t);
                }
                Ms += (size_t)TS * N * NP;          // S.S follows S in the buffer
            }
            if (has_work && (kind == 1 || K > 1) && !(a.ablate & 1)) {
                const uint32_t tap_off = (kind == 0 ? 1u : 2u) * L.a_unit;
                {
                    float4 zh[NA];
                    gp_propagate_half<N, 0, NA, 0>(Ms, xv, zh);
                    if (st_ok) gp_store_rows<N, 0, NA>(ahi0, tap_off, zh);
                }
                if (NB > 0) {
                    float4 zh[NB > 0 ? NB : 1];
                    gp_propagate_half<N, NA, (NB > 0 ? NB : 1), SLOT_B>(Ms, xv, zh);
                    if (st_ok) gp_store_rows<N, NA, (NB > 0 ? NB : 1)>(ahi0, tap_off, zh);
                }
            }
            fence_proxy_async_smem();       // st.shared operand rows -> visible to the tensor cores
            __syncwarp();
            if (lane == 0) gp_arrive(&a_full[slot]);
            if (TIMING) {
                tm[2] += (unsigned long long)(clock64() - t_item0);
                tm[3] += 1;
            }
        }
        if (cur_tile >= 0) {
            __syncwarp();
            if (lane == 0) gp_arrive(&s_free[cur_tile & 1]);
        }
        if (TIMING && a.timing && lane == 0 && warp == 0) {
            atomicAdd(&a.timing[0], tm[0]); atomicAdd(&a.timing[1], tm[1]); atomicAdd(&a.timing[2], tm[2]);
            atomicAdd(&a.timing[3], tm[3]);
        }
    }
    if (TIMING && a.timing && tid == 0) {
        atomicAdd(&a.timing[12], (unsigned long long)(clock64() - t_kernel0));
        atomicAdd(&a.timing[14], 1ull);
    }
}

// ---------------------------------------------------------------------------------------
// tap images: w [F][1][K][G] -> K*4 units (chunk-major: the K units of one 32-feature chunk are contiguous) of 128 rows x
// 128 bytes [hi 32 | lo 32] fp16 of w * 2^e, SWIZZLE_128B K-major; e from the largest |w| so that |w| * 2^e < 2^15
// ---------------------------------------------------------------------------------------
// largest |w| over the taps: one value per thread, block maximum, atomicMax on the (non-negative) float bits
__global__ void __launch_bounds__(1024) gp_tap_absmax_kernel(const float* __restrict__ w, int n, unsigned int* __restrict__ maxbits) {
    __shared__ float red[32];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float mx = i < n ? fabsf(w[i]) : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = red[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (threadIdx.x == 0) atomicMax(maxbits, __float_as_uint(mx));
    }
}
// 2^e with |w|max * 2^e < 2^15 (and its inverse)
__device__ __forceinline__ void gp_scale_from_max(float mx, float& s, float& si) {
    s = 1.f;
    si = 1.f;
    const int q = (int)((__float_as_uint(mx) >> 23) & 0xFF) - 127;
    if (mx > 0.f && q < 128) {
        const int e = max(-100, min(100, 14 - q));
        s = __uint_as_float((uint32_t)(e + 127) << 23);
        si = __uint_as_float((uint32_t)(127 - e) << 23);
    }
}

__global__ void gp_prep_taps_kernel(const float* __restrict__ w, unsigned char* __restrict__ img,
                                    float* __restrict__ wscale, int K) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;     // one (f, k, g) element each
    float sc, sci;
    gp_scale_from_max(__uint_as_float(reinterpret_cast<const unsigned int*>(wscale)[2]), sc, sci);
    if (idx == 0) {
        wscale[0] = sc;         // read by the filter kernel's epilogue
        wscale[1] = sci;
    }
    if (idx >= GP_C * K * GP_C) return;
    const int f = idx / (K * GP_C), kg = idx - f * (K * GP_C), k = kg / GP_C, gch = kg - k * GP_C;
    const int c = gch >> 5, l = gch & 31;
    const float v = w[idx] * sc;
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    unsigned char* unit = img + (size_t)(c * K + k) * GP_BUNIT;
    *reinterpret_cast<__half*>(unit + sw128_offset(f, l >> 3) + (l & 7) * 2) = hi;
    *reinterpret_cast<__half*>(unit + sw128_offset(f, 4 + (l >> 3)) + (l & 7) * 2) = lo;
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
size_t gf_pair_image_bytes(int K) { return (size_t)K * GP_NCHUNK * GP_BUNIT + 64; }   // + {scale, 1/scale}

// (the producer schedule assumes at most one item per warp per group: ceil(128 / N / 4) <= 8 producer warps)
bool gf_pair_supported(int N, int K) { return N == 10 && K >= 1 && K <= GP_MAX_K; }

int launch_prep_pair_taps(const float* w, void* img, int K, cudaStream_t st) {
    unsigned char* base = reinterpret_cast<unsigned char*>(img);
    float* wscale = reinterpret_cast<float*>(base + (size_t)K * GP_NCHUNK * GP_BUNIT);
    const int n = GP_C * K * GP_C;
    GPP_CUDA_OK(cudaMemsetAsync(wscale, 0, 16, st));
    gp_tap_absmax_kernel<<<(n + 1023) / 1024, 1024, 0, st>>>(w, n, reinterpret_cast<unsigned int*>(wscale) + 2);
    GPP_LAUNCH_CHECK();
    gp_prep_taps_kernel<<<(n + 255) / 256, 256, 0, st>>>(w, base, wscale, K);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

static unsigned long long* g_pair_timing = nullptr;   // "tc_timing" debug counters

// wa_host / ba_host: HOST copies of the action MLP (they travel as kernel parameters), or null
int launch_gf_forward_pair(const float* x, const void* S, int s_is_f64, const void* wimg, const float* bias, float* y,
                           const float* wa_host, const float* ba_host, float* logits, int B, int N, int K, int relu,
                           cudaStream_t st) {
    GPP_REQUIRE(gf_pair_supported(N, K), GPP_ERR_UNSUPPORTED, "gf_forward_pair: N=%d K=%d outside the pair kernel's envelope", N, K);
    GPP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (reinterpret_cast<uintptr_t>(y) & 15u) == 0, GPP_ERR_INVALID,
                "gf_forward_pair: x and y must be 16-byte aligned");
    GPP_REQUIRE((wa_host != nullptr) == (logits != nullptr), GPP_ERR_INVALID, "gf_forward_pair: logits need the action MLP");
    static GpArgs a;       // large (kernel-parameter image); filled per call, copied by the launch
    static_assert(sizeof(GpArgs) <= 4096, "kernel parameters exceed 4 KB");
    const int TS = GP_M / N;
    a.x = x; a.S = S;
    a.wimg = reinterpret_cast<const unsigned char*>(wimg);
    a.wscale = reinterpret_cast<const float*>(a.wimg + (size_t)K * GP_NCHUNK * GP_BUNIT);
    a.bias = bias; a.y = y; a.logits = logits;
    a.B = B; a.K = K; a.TS = TS;
    a.num_tiles = (B + TS - 1) / TS;
    a.s_is_f64 = s_is_f64; a.relu = relu; a.has_act = wa_host ? 1 : 0;
    a.ablate = debug_option(DBG_PAIR_ABLATE);
    a.timing = nullptr;
    if (debug_option(DBG_TC_TIMING)) {
        if (!g_pair_timing) {
            GPP_CUDA_OK(cudaMalloc(&g_pair_timing, 128));
            GPP_CUDA_OK(cudaMemset(g_pair_timing, 0, 128));
        }
        a.timing = g_pair_timing;
    }
    if (wa_host) {
        for (int i = 0; i < GP_ACT * GP_C; ++i) a.wa[i] = wa_host[i];
        for (int i = 0; i < GP_ACT; ++i) a.ba[i] = ba_host[i];
    }
    const size_t smem = GpSmem(N, K, TS).total;
    GPP_REQUIRE(smem <= 227 * 1024, GPP_ERR_UNSUPPORTED, "gf_forward_pair: %zu bytes of shared memory do not fit", smem);
    static SmemConfig smem_cfg, smem_cfg_t;
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    if (a.timing) {
        GPP_CUDA_OK(ensure_dynamic_smem(gf_fwd_pair_kernel<10, true>, smem_cfg_t, smem));
        gf_fwd_pair_kernel<10, true><<<grid, GP_THREADS, smem, st>>>(a);
    } else {
        GPP_CUDA_OK(ensure_dynamic_smem(gf_fwd_pair_kernel<10, false>, smem_cfg, smem));
        gf_fwd_pair_kernel<10, false><<<grid, GP_THREADS, smem, st>>>(a);
    }
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp

// debug: per-role cycle totals of gf_fwd_pair_kernel since the last call (filled only with the "tc_timing" option):
// [0..3] producer warp 0: wait S, wait ring slot, item work, items; [4] MMA warpgroup: wait operands, [6] its loop
// total, [8] its epilogue work; [9..10] scout: wait S buffer, work; [11] tiles; [12] kernel cycles (thread 0 of every
// CTA); [14] CTAs
extern "C" int gpp_debug_pair_timing(unsigned long long* out16) {
    if (!gpp::g_pair_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out16, gpp::g_pair_timing, 128, cudaMemcpyDeviceToHost);
    cudaMemset(gpp::g_pair_timing, 0, 128);
    return GPP_OK;
}
