// im2col-free tensor-core feature extractor (Hopper wgmma): the per-agent CNN + compress MLP of DecentralPlannerNet
// (reference graphs/models/decentralplanner.py:155-195,284-290, eval mode) with fp16 2-way split operands (fp32
// parity), 8 agents per tile, one persistent CTA per SM.
//
// Layout idea.  An activation map lives in shared memory as fp16 (hi | lo) planes of 8 channels, one 16-byte vector per
// padded pixel, pixels in ONE linear order over the whole tile:   row = y * (8 agents * Wp) + agent * Wp + x.
// That is exactly the canonical NO-SWIZZLE K-major operand layout of a wgmma descriptor (rows 16 B apart, 8-row groups
// 128 B apart, K planes `rows * 16` B apart), and in it the 3x3 tap (ky, kx) of EVERY output pixel is the same buffer
// shifted by (ky * 8 * Wp + kx) rows: the A operand of a tap is just the descriptor start address moved by a multiple
// of 16 B.  No im2col copy exists anywhere: an epilogue writes a layer's output once, and the next layer's 9 taps x
// Cin/16 MMAs read it in place.  With the y-major order the rows a layer needs (y < Hout) are a prefix, so M covers
// needed image rows only.
//
//   layer  in grid (Hp x Wp)  rows   planes  out ch  M tiles  taps x k16   B bytes
//   conv0  13 x 16 (11+pad)   1664   1       32      10       3 x 2 (*)    6 KB    (*) two ky taps per K=16: LBO = one row;
//                                                                               W_hi and W_lo share the 8-channel K slot
//   conv1  7 x 7              392    4       32      3        9 x 2        36 KB
//   conv2  7 x 8              448    4       64      2        9 x 2        72 KB
//   conv3  4 x 4              128    8       64      1        9 x 4        144 KB
//   conv4  4 x 4              128    8       128     1        9 x 4        288 KB
//   linear 1 x 1              8      16      128     1        1 x 8        64 KB
//
// Precision: v = hi + lo with hi = fp16(v * 2^e), lo = fp16(v * 2^e - hi); products hi*hi + lo*hi + hi*lo accumulate
// in fp32 registers.  e is chosen per agent and layer from the running maximum (two-pass epilogue),
// weights are scaled per layer; residual ~2^-22 per product.  Each K plane of a filter image holds, per warpgroup's
// channel group, [W_hi | W_lo] rows side by side, so A_hi x (W_hi, W_lo) is ONE MMA of twice the width and A_lo x W_hi
// a second; the hi.lo half of the accumulator is added to the rest after the layer.
//
// Roles: warps 0-7 = two warpgroups.  conv0..conv2 (several 64-row blocks) split the rows: warpgroup h computes block h
// of every 128-row M tile for all output channels; conv3, conv4 and the linear layer (one block) split the channels.
// Each warpgroup issues its wgmma (M = 64 per instruction; a chunk's ring slot is released one chunk later, so the
// MMAs stream), stages its accumulators through shared memory and runs the epilogue (BatchNorm/ReLU/max-pool -> fp16
// split -> next layer's operand buffer); warps 8-11 = loader warpgroup, one lane of which streams filter chunks
// through a 5 x 16 KB ring of bulk copies and the input tiles; it gives its registers to the compute warpgroups.
#include "common.cuh"
#include "feature.cuh"
#include "tc_common.cuh"

#include <cuda_fp16.h>
#include <stdio.h>

namespace gpp {

constexpr int FM_A = 8;                        // agents per tile
constexpr int FM_EPI_WARPS = 8;
constexpr int FM_EPI_THREADS = 32 * FM_EPI_WARPS;
constexpr int FM_LOADER_WARP = FM_EPI_WARPS;
constexpr int FM_THREADS = FM_EPI_THREADS + 128;   // + a loader warpgroup, of which one lane works (setmaxnreg)
constexpr int FM_LOADER_REGS = 40, FM_EPI_REGS = 232;  // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int FM_SLOTS = 5, FM_SLOT_BYTES = 16384;
constexpr int FM_NL = 6;

__host__ __device__ constexpr int fm_n(int L) { return L < 2 ? 32 : L < 4 ? 64 : 128; }
__host__ __device__ constexpr int fm_wp(int L) { return L == 0 ? 16 : L == 1 ? 7 : L == 2 ? 8 : L < 5 ? 4 : 1; }
__host__ __device__ constexpr int fm_hp(int L) { return L == 0 ? 13 : L < 3 ? 7 : L < 5 ? 4 : 1; }
__host__ __device__ constexpr int fm_aw(int L) { return FM_A * fm_wp(L); }
__host__ __device__ constexpr int fm_rows(int L) { return fm_hp(L) * fm_aw(L); }
__host__ __device__ constexpr int fm_planes(int L) { return L == 0 ? 1 : L < 3 ? 4 : L < 5 ? 8 : 16; }
__host__ __device__ constexpr int fm_lbo(int L) { return fm_rows(L) * 16; }
__host__ __device__ constexpr int fm_tiles(int L) { return L == 0 ? 10 : L == 1 ? 3 : L == 2 ? 2 : 1; }
__host__ __device__ constexpr int fm_hout(int L) { return L == 0 ? 10 : L == 1 ? 5 : L == 2 ? 4 : L < 5 ? 2 : 1; }
__host__ __device__ constexpr int fm_ks(int L) { return L < 3 ? 2 : L < 5 ? 4 : 8; }           // K=16 steps per tap
__host__ __device__ constexpr int fm_taps(int L) { return L == 5 ? 1 : 9; }
__host__ __device__ constexpr int fm_units(int L) { return L == 0 ? 1 : fm_taps(L) * fm_ks(L); }
__host__ __device__ constexpr int fm_unit_bytes(int L) { return L == 0 ? 6144 : L < 4 ? 64 * fm_n(L) : 8192; }
__host__ __device__ constexpr int fm_upc(int L) { return L == 0 ? 1 : L == 1 ? 8 : L < 4 ? 4 : 2; }   // units per chunk
__host__ __device__ constexpr int fm_chunks(int L) { return (fm_units(L) + fm_upc(L) - 1) / fm_upc(L); }
__host__ __device__ constexpr int fm_img_bytes(int L) { return fm_units(L) * fm_unit_bytes(L); }
// Work split between the two warpgroups.  conv0..conv2 have several 64-row blocks per 128-row M tile: warpgroup h takes
// block h of every M tile for ALL output channels, so each A row is read by one warpgroup only.  conv3, conv4 and the
// linear layer have one block: warpgroup h takes half h of the output channels.
__host__ __device__ constexpr bool fm_rowsplit(int L) { return L <= 2; }
__host__ __device__ constexpr int fm_nc(int L) { return fm_rowsplit(L) ? fm_n(L) : fm_n(L) / 2; }     // channels per WG
// Layers 1..5 issue A_hi x [W_hi | W_lo] as one MMA of width 2 NC (the W_lo half of the accumulator is added to the
// W_hi half after the layer), then A_lo x W_hi: two instructions per product instead of three.
__host__ __device__ constexpr int fm_af(int L) { return fm_nc(L); }     // accumulator floats per 64-row block

// shared-memory map (bytes from the 1024-aligned base)
constexpr int FM_R1 = 0;                           // in0 (hi|lo) -> act2 -> act4
constexpr int FM_R1_BYTES = 57344;
constexpr int FM_R2 = FM_R1 + FM_R1_BYTES;         // act1 -> act3 -> act5
constexpr int FM_R2_BYTES = 50176;
constexpr int FM_XRAW = FM_R2 + FM_R2_BYTES;       // raw fp32 inputs of the tile (bulk copy target)
constexpr int FM_XRAW_BYTES = 11648;
constexpr int FM_STG = FM_XRAW + FM_XRAW_BYTES;    // pooling partners that live in another warp
constexpr int FM_STG_BYTES = 8192;
constexpr int FM_RING = FM_STG + FM_STG_BYTES;
constexpr int FM_CST = FM_RING + FM_SLOTS * FM_SLOT_BYTES;      // epilogue constants [L][scale | shift][128] floats
constexpr int FM_CST_BYTES = 6 * 2 * 128 * 4;
constexpr int FM_MISC = FM_CST + FM_CST_BYTES;
constexpr int FM_SMEM_BYTES = FM_MISC + 1024;
static_assert(2 * fm_planes(0) * fm_lbo(0) <= FM_R1_BYTES && 2 * fm_planes(2) * fm_lbo(2) <= FM_R1_BYTES, "R1");
static_assert(2 * fm_planes(1) * fm_lbo(1) <= FM_R2_BYTES && 2 * fm_planes(3) * fm_lbo(3) <= FM_R2_BYTES, "R2");
static_assert(FM_SMEM_BYTES <= 232448, "shared memory budget");
__host__ __device__ constexpr int fm_in_base(int L) { return (L == 0 || L == 2 || L == 4) ? FM_R1 : FM_R2; }

struct FmMisc {
    uint64_t w_full[FM_SLOTS], w_free[FM_SLOTS];
    uint64_t xraw_full, xraw_free;
    uint32_t xflag;                    // tile has a non-zero lo part in its inputs
    uint32_t amax[FM_NL][FM_A];        // running max (float bits, values >= 0) of layer L's output per agent
    float mul0[FM_A], inv0[FM_A];      // input scale 2^e0 and its inverse
    float mul1[FM_A], inv1[FM_A];      // act1 scale (from the weight-norm bound of conv0) and its inverse
};
static_assert(sizeof(FmMisc) <= 1024, "misc block");

// constants block in global memory (floats): [L][0][c] = epilogue scale, [L][1][c] = shift; then misc
constexpr int FM_CONST_MISC = FM_NL * 2 * 128;
constexpr int FM_CONST_FLOATS = FM_CONST_MISC + 16;

struct FmArgs {
    const float* x;
    float* feat;
    int total_agents, num_tiles;
    const unsigned char* img[FM_NL];
    const float* consts;
    int x_bulk;     // the inputs may be fetched with bulk copies (device memory, 16-byte aligned)
    int pdl;
    unsigned long long* timing;
};

// ---- waits -------------------------------------------------------------------------------------------------------
constexpr long long FM_WATCHDOG_CYCLES = 2000000000LL;
__device__ __forceinline__ bool fm_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(1000000u)
        : "memory");
    return ok != 0;
}
// Watchdog: a barrier that does not complete within ~1 s traps instead of hanging the GPU.  No printf: a function call
// anywhere in the kernel makes ptxas serialise its wgmma pipelines.
__device__ __forceinline__ void fm_wait(uint64_t* bar, uint32_t parity) {
    if (fm_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!fm_try_wait(bar, parity))
        if (clock64() - t0 > FM_WATCHDOG_CYCLES) __trap();
}
__device__ __forceinline__ void fm_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fm_arrive_warp(uint64_t* bar) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) fm_arrive(bar);
}
__device__ __forceinline__ void fm_epi_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// scale exponent for a running maximum m >= 0 (float bits): m * 2^e in [2^9, 2^10)
__device__ __forceinline__ int fm_scale_exp(uint32_t bits) {
    if (bits == 0) return 0;
    int e = 9 - ((int)(bits >> 23) - 127);
    return e < -110 ? -110 : (e > 110 ? 110 : e);
}
__device__ __forceinline__ float fm_pow2(int e) { return __int_as_float((e + 127) << 23); }

// 8 floats -> 8 x fp16 hi (16 B) and 8 x fp16 lo
__device__ __forceinline__ void fm_split8(const float* v, uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __half2 hh = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        const float2 f = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(v[2 * i] - f.x, v[2 * i + 1] - f.y);
        h[i] = *reinterpret_cast<const uint32_t*>(&hh);
        l[i] = *reinterpret_cast<const uint32_t*>(&ll);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ void fm_sts16(uint32_t addr, const uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// debug phase timers (A.timing != null): 6-11 wait-for-filters per layer, 12-17 MMA per layer, 18 tiles, 19 convert,
// 26-31 epilogue work per layer (warp 0 of block 0)
// tacc = the debug buffer in the one thread that records (thread 0 of block 0), null everywhere else
#define FM_T0() const long long _t0 = tacc ? clock64() : 0
#define FM_ACC(slot) do { if (tacc) atomicAdd(&tacc[slot], (unsigned long long)(clock64() - _t0)); } while (0)

// ring position of the next filter chunk (the same sequence the loader fills)
struct FmRing {
    uint32_t slot, phase;
    __device__ __forceinline__ void advance() { if (++slot == FM_SLOTS) { slot = 0; phase ^= 1; } }
};
__device__ __forceinline__ uint64_t fm_desc(uint32_t addr, uint32_t lbo) { return gmma_desc_nosw(addr, lbo, 128); }

// ---- MMAs of one layer L >= 1 for warpgroup h: acc[t] = rows t * 128 + (row split ? 64 h : 0) .. + 63 of the layer's
//      M tiles, fm_nc(L) channels (after the layer, the first fm_nc(L) / 2 floats).  Every descriptor offset but the
//      warpgroup's own is a compile-time constant (fully unrolled).  A chunk's ring slot is freed once the MMAs of the
//      NEXT chunk are issued (wait_group 1), so the tensor pipe does not drain at every chunk.
template <int L>
__device__ __forceinline__ void fm_mma_layer(uint32_t sm_base, FmMisc* ms, FmRing& ring, int h, float (&acc)[fm_tiles(L)][fm_af(L)],
                                             unsigned long long* tacc) {
    constexpr int NC = fm_nc(L), KS = fm_ks(L), UNITS = fm_units(L), UPC = fm_upc(L), UB = fm_unit_bytes(L);
    constexpr int AW = fm_aw(L), LBO = (L == 5) ? 128 : fm_lbo(L), TILES = fm_tiles(L);
    constexpr uint32_t A_HI = fm_in_base(L), A_LO = fm_in_base(L) + fm_planes(L) * LBO;
    constexpr int CHUNKS = fm_chunks(L);
    // B planes of 2N rows; this warpgroup's NC channels are [W_hi NC rows | W_lo NC rows] in them (fm_prep_image_kernel)
    constexpr uint32_t BLBO = 32 * fm_n(L);
    const uint32_t b_off = fm_rowsplit(L) ? 0u : (uint32_t)(h * 2 * NC * 16);
    const uint32_t a_off = fm_rowsplit(L) ? (uint32_t)(h * 64 * 16) : 0u;
    uint32_t prev = 0;
#pragma unroll
    for (int cc = 0; cc < CHUNKS; ++cc) {
        {
            FM_T0();
            fm_wait(&ms->w_full[ring.slot], ring.phase);
            FM_ACC(6 + L);
        }
        FM_T0();
        const uint32_t bs = sm_base + FM_RING + ring.slot * FM_SLOT_BYTES + b_off;
        const uint32_t as = sm_base + a_off;
        wgmma_fence();
#pragma unroll
        for (int uu = 0; uu < UPC; ++uu) {
            const int u = cc * UPC + uu;
            if (u < UNITS) {
                const int tap = u / KS, k16 = u - tap * KS;
                const int shift = (L == 5) ? 0 : ((tap / 3) * AW + (tap % 3));
                const uint64_t db = fm_desc(bs + uu * UB, BLBO);
#pragma unroll
                for (int t = 0; t < TILES; ++t) {
                    const uint32_t aoff = (uint32_t)((t * 128 + shift) * 16 + k16 * 2 * LBO);
                    wgmma_f16<2 * NC>(acc[t], fm_desc(as + A_HI + aoff, LBO), db, u > 0);
                    wgmma_f16<NC>(acc[t], fm_desc(as + A_LO + aoff, LBO), db, 1);
                }
            }
        }
        wgmma_commit();
        if (cc > 0) {
            wgmma_wait<1>();
            fm_arrive_warp(&ms->w_free[prev]);
        }
        prev = ring.slot;
        ring.advance();
        FM_ACC(12 + L);
    }
    {
        FM_T0();
        wgmma_wait<0>();
        fm_arrive_warp(&ms->w_free[prev]);
        FM_ACC(12 + L);
    }
#pragma unroll
    for (int t = 0; t < TILES; ++t)
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) acc[t][i] += acc[t][i + NC / 2];
}

// ---- epilogue pieces -----------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 fm_lds4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// 16 output channels of this thread's accumulator row: acc * (scale * inv) + shift, ReLU.  src = the staged accumulator
// of the first channel, cs = shared-memory constants of the first channel ([0..] scale, [128..] shift)
__device__ __forceinline__ void fm_block_vals(const float* src, const float* cs, float inv, float (&u)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
        const float4 a = fm_lds4(src + i);
        const float4 sc = fm_lds4(cs + i), sh = fm_lds4(cs + 128 + i);
        u[i] = fmaxf(fmaf(a.x, sc.x * inv, sh.x), 0.f);
        u[i + 1] = fmaxf(fmaf(a.y, sc.y * inv, sh.y), 0.f);
        u[i + 2] = fmaxf(fmaf(a.z, sc.z * inv, sh.z), 0.f);
        u[i + 3] = fmaxf(fmaf(a.w, sc.w * inv, sh.w), 0.f);
    }
}
__device__ __forceinline__ float fm_max16(const float (&u)[16]) {
    float m0 = fmaxf(u[0], u[1]), m1 = fmaxf(u[2], u[3]), m2 = fmaxf(u[4], u[5]), m3 = fmaxf(u[6], u[7]);
#pragma unroll
    for (int i = 8; i < 16; i += 4) {
        m0 = fmaxf(m0, u[i]); m1 = fmaxf(m1, u[i + 1]); m2 = fmaxf(m2, u[i + 2]); m3 = fmaxf(m3, u[i + 3]);
    }
    return fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
}
// 2-wide max-pool along x between the lanes of a pair (even lane = even x): afterwards the even lane holds the pooled
// channels 0-7 of the block and the odd lane channels 8-15 -- half the shuffles of a full exchange, and both lanes store
__device__ __forceinline__ void fm_xpool(const float (&u)[16], int odd, float (&p)[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float send = odd ? u[i] : u[i + 8];
        const float mine = odd ? u[i + 8] : u[i];
        p[i] = fmaxf(mine, __shfl_xor_sync(0xffffffffu, send, 1));
    }
}
// store 8 scaled channels as one (hi, lo) pair of 16-byte vectors in plane `plane` of the buffer at `base`
__device__ __forceinline__ void fm_store8(uint32_t base, int lbo, int planes, int row, int plane, const float (&p)[8], float mul) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = p[i] * mul;
    uint4 hi, lo;
    fm_split8(v, hi, lo);
    const uint32_t addr = base + plane * lbo + row * 16;
    fm_sts16(addr, hi);
    fm_sts16(addr + planes * lbo, lo);
}
__device__ __forceinline__ void fm_zero(uint32_t addr, int bytes, int et) {
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int i = et * 16; i < bytes; i += FM_EPI_THREADS * 16) fm_sts16(addr + i, z);
}

// row stride (floats) of an accumulator tile staged in shared memory: padded against bank conflicts of row-per-lane reads
__host__ __device__ constexpr int fm_srow(int L) { return fm_n(L) + 4; }

// layers 1..5: MMAs into registers; per M tile the accumulators are staged (rows x fm_srow floats) in the layer's INPUT
// buffer, which no MMA reads any more.  Dynamic-scale layers 1..4 then run pass 1 = values (kept in registers) +
// per-agent maximum (+ pooling partners that live in another warp go through FM_STG), pass 2 = scale, split, store.
template <int L>
__device__ __forceinline__ void fm_epilogue_dyn(unsigned char* sm, uint32_t sm_base, FmMisc* ms, FmRing& ring, int na,
                                                int q, int h, int lane, int et, unsigned long long* tacc) {
    constexpr int N = fm_n(L), AW = fm_aw(L), WP = fm_wp(L), HO = fm_hout(L), TILES = fm_tiles(L);
    constexpr bool POOL = (L == 2 || L == 4);
    constexpr int LO = L + 1;                                      // the layer that consumes the output
    constexpr uint32_t OUT = fm_in_base(LO);
    constexpr int OLBO = (LO == 5) ? 128 : fm_lbo(LO), OPL = fm_planes(LO), OAW = fm_aw(LO), OWP = fm_wp(LO);
    constexpr int NB = N / 32;                                     // 16-channel blocks per thread (channel half h)
    constexpr int CV = POOL ? 8 : 16;
    constexpr int SROW = fm_srow(L);
    const int wt = et & 127;                                       // thread of the warpgroup
    float acc[TILES][fm_af(L)];
    fm_mma_layer<L>(sm_base, ms, ring, h, acc, tacc);
    fm_epi_sync();                                                 // both warpgroups' MMAs are done with the input buffer
    FM_T0();
    fm_zero(sm_base + OUT, (LO == 5) ? 8192 : 2 * OPL * OLBO, et);
    float* sacc = reinterpret_cast<float*>(sm + fm_in_base(L));
    float* stg = reinterpret_cast<float*>(sm + FM_STG);
    const float* cs = reinterpret_cast<const float*>(sm + FM_CST) + L * 256 + h * (N / 2);
    const int l = q * 32 + lane, odd = lane & 1;
    const bool rows_here = (L == 1 || L == 2) ? true : (q < 2);     // conv3 / conv4: the valid rows are lanes 0..63
    const bool upper = (L == 2) ? (q >= 2) : (q == 1);              // pooled layers: rows whose y is odd
    float cv[TILES][NB][CV];
#pragma unroll
    for (int t = 0; t < TILES; ++t) {
        if (t > 0) fm_epi_sync();                                   // pass 1 of tile t - 1 has read the staging buffer
#pragma unroll
        for (int i = 0; i < fm_nc(L) / 2; i += 2) {
            const int row = (fm_rowsplit(L) ? 64 * h : 0) + wg_row(wt, i);
            const int col = (fm_rowsplit(L) ? 0 : h * (N / 2)) + wg_col(wt, i);
            *reinterpret_cast<float2*>(sacc + row * SROW + col) = make_float2(acc[t][i], acc[t][i + 1]);
        }
        fm_epi_sync();
        if (rows_here) {
            const int r = t * 128 + l;
            const int y = r / AW, a = (r % AW) / WP, x = r % WP;
            const bool valid = y < HO && x < HO && a < na;
            const float inv = (L == 1) ? ms->inv1[a] : fm_pow2(-fm_scale_exp(ms->amax[L - 1][a]));
            float mx = 0.f;
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                float u[16];
                fm_block_vals(sacc + l * SROW + h * (N / 2) + 16 * b, cs + 16 * b, inv, u);
                mx = fmaxf(mx, fm_max16(u));
                if constexpr (POOL) {
                    fm_xpool(u, odd, cv[t][b]);
                    if (upper && valid) {        // the y partner lives 64 (conv2) / 32 (conv4) lanes down: park the values
                        float* dst = stg + (((L == 2 ? t * FM_A + a : a) * (L == 2 ? 2 : 1) + (x >> 1)) * N + h * (N / 2) + 16 * b + 8 * odd);
                        *reinterpret_cast<float4*>(dst) = make_float4(cv[t][b][0], cv[t][b][1], cv[t][b][2], cv[t][b][3]);
                        *reinterpret_cast<float4*>(dst + 4) = make_float4(cv[t][b][4], cv[t][b][5], cv[t][b][6], cv[t][b][7]);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) cv[t][b][i] = u[i];
                }
            }
            if (valid) atomicMax(&ms->amax[L][a], __float_as_uint(mx));
        }
    }
    fm_epi_sync();
    const bool writer = POOL ? (rows_here && !upper) : rows_here;
    if (writer) {
#pragma unroll
        for (int t = 0; t < TILES; ++t) {
            const int r = t * 128 + l;
            const int y = r / AW, a = (r % AW) / WP, x = r % WP;
            const bool valid = y < HO && x < HO && a < na;
            const float mul = fm_pow2(fm_scale_exp(ms->amax[L][a]));
            int orow;
            if (LO == 5) orow = a;
            else if (POOL) orow = ((y >> 1) + 1) * OAW + a * OWP + (x >> 1) + 1;
            else orow = (y + 1) * OAW + a * OWP + x + 1;
            if (valid) {
#pragma unroll
                for (int b = 0; b < NB; ++b) {
                    const int c0 = h * (N / 2) + 16 * b;
                    if constexpr (POOL) {
                        const float* src = stg + (((L == 2 ? t * FM_A + a : a) * (L == 2 ? 2 : 1) + (x >> 1)) * N + c0 + 8 * odd);
                        const float4 p0 = fm_lds4(src), p1 = fm_lds4(src + 4);
                        float p[8];
                        p[0] = fmaxf(cv[t][b][0], p0.x); p[1] = fmaxf(cv[t][b][1], p0.y);
                        p[2] = fmaxf(cv[t][b][2], p0.z); p[3] = fmaxf(cv[t][b][3], p0.w);
                        p[4] = fmaxf(cv[t][b][4], p1.x); p[5] = fmaxf(cv[t][b][5], p1.y);
                        p[6] = fmaxf(cv[t][b][6], p1.z); p[7] = fmaxf(cv[t][b][7], p1.w);
                        fm_store8(sm_base + OUT, OLBO, OPL, orow, (c0 >> 3) + odd, p, mul);
                    } else {
                        float p[8];
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                            for (int i = 0; i < 8; ++i) p[i] = cv[t][b][8 * hh + i];
                            fm_store8(sm_base + OUT, OLBO, OPL, orow, (c0 >> 3) + hh, p, mul);
                        }
                    }
                }
            }
        }
    }
    fence_proxy_async_smem();              // st.shared operand rows -> visible to the next layer's wgmma
    fm_epi_sync();
    FM_ACC(26 + L);
}

// conv0 MMAs of image rows 2j, 2j + 1 (acc[tt]) for the 64-row block that starts at a_hi, all 32 channels; LO: the
// inputs are not fp16-exact, add their lo planes.  The choice is made outside the instruction sequence: a branch
// between two wgmma makes the compiler serialise them.
template <bool LO>
__device__ __forceinline__ void fm_conv0_mma(float (&acc)[2][16], uint32_t a_hi, uint32_t bs, int j) {
    wgmma_fence();
#pragma unroll
    for (int tt = 0; tt < 2; ++tt) {
        const uint32_t arow = (uint32_t)((2 * j + tt) * 128);      // rows of 16 bytes
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
            for (int pr = 0; pr < 2; ++pr) {        // K = 16 = image rows ky = 2 pr, 2 pr + 1 (LBO = one row)
                const uint32_t aoff = (arow + 2 * pr * 128 + kx) * 16;
                const uint64_t db = fm_desc(bs + (kx * 2 + pr) * 1024, 512);
                wgmma_f16<32>(acc[tt], fm_desc(a_hi + aoff, 2048), db, (kx | pr) != 0);
                if constexpr (LO) wgmma_f16<32>(acc[tt], fm_desc(a_hi + fm_lbo(0) + aoff, 2048), db, 1);
            }
    }
    wgmma_commit();
}

// =====================================================================================================================
__global__ void __launch_bounds__(FM_THREADS, 1) feature_mma_kernel(const FmArgs A) {
    extern __shared__ __align__(1024) unsigned char sm[];
    FmMisc* ms = reinterpret_cast<FmMisc*>(sm + FM_MISC);
    const uint32_t sm_base = smem_u32(sm);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < FM_SLOTS; ++s) { mbar_init(&ms->w_full[s], 1); mbar_init(&ms->w_free[s], FM_EPI_WARPS); }
        mbar_init(&ms->xraw_full, 1);
        mbar_init(&ms->xraw_free, FM_EPI_WARPS);
        fence_mbar_init();
    }
    __syncthreads();
    const float* __restrict__ cst = A.consts;
    unsigned long long* tacc = (blockIdx.x == 0 && threadIdx.x == 0) ? A.timing : nullptr;
    griddep_launch_dependents();       // the next kernel of the stream may start its prologue; it still waits for this grid

    if (warp >= FM_LOADER_WARP) {
        // ================= loader =================
        // Its warpgroup hands its registers to the compute warpgroups: with a lone 9th warp instead, 3 warps share one
        // SM sub-partition and every thread is capped at 168 registers, which made the epilogues spill.
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FM_LOADER_REGS));
        if (warp == FM_LOADER_WARP && lane == 0) {
            uint32_t g = 0;
            int it = 0;
            auto issue_x = [&](int tile) {
                const int na = min(FM_A, A.total_agents - tile * FM_A);
                if (A.x_bulk && na == FM_A) {
                    mbar_arrive_expect_tx(&ms->xraw_full, FM_A * 363 * 4);
                    bulk_g2s(sm + FM_XRAW, A.x + (size_t)tile * FM_A * 363, FM_A * 363 * 4, &ms->xraw_full);
                } else {
                    fm_arrive(&ms->xraw_full);        // the compute warps read this tile straight from global memory
                }
            };
            for (int tile = blockIdx.x; tile < A.num_tiles; tile += gridDim.x, ++it) {
                int c = 0;
                for (int L = 0; L < FM_NL; ++L) {
                    const int nch = fm_chunks(L), upc = fm_upc(L), ub = fm_unit_bytes(L), units = fm_units(L);
                    for (int cc = 0; cc < nch; ++cc, ++c, ++g) {
                        if (it == 0 && c == FM_SLOTS - 1) {
                            if (A.pdl) griddep_wait();
                            issue_x(tile);
                        }
                        if (c == 8) {
                            const int next = tile + gridDim.x;
                            if (next < A.num_tiles) {
                                fm_wait(&ms->xraw_free, it & 1);
                                issue_x(next);
                            }
                        }
                        const uint32_t slot = g % FM_SLOTS, use = g / FM_SLOTS;
                        if (use >= 1) fm_wait(&ms->w_free[slot], (use - 1) & 1);
                        const int nu = (units - cc * upc) < upc ? (units - cc * upc) : upc;
                        const uint32_t bytes = (uint32_t)(nu * ub);
                        mbar_arrive_expect_tx(&ms->w_full[slot], bytes);
                        bulk_g2s(sm + FM_RING + slot * FM_SLOT_BYTES, A.img[L] + (size_t)cc * upc * ub, bytes,
                                 &ms->w_full[slot]);
                    }
                }
            }
        }
    } else {
        // ================= compute warps: two warpgroups (fm_rowsplit: row blocks or channel halves h) =================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FM_EPI_REGS));
        const int q = warp & 3, h = warp >> 2, et = threadIdx.x, wt = et & 127;
        FmRing ring;
        ring.slot = 0; ring.phase = 0;
        int it = 0;
        if (A.pdl) griddep_wait();         // x (and the feature buffer's previous readers) belong to earlier kernels
        for (int tile = blockIdx.x; tile < A.num_tiles; tile += gridDim.x, ++it) {
            const int na = min(FM_A, A.total_agents - tile * FM_A);
            const bool bulk = A.x_bulk && na == FM_A;
            // ---- inputs: per-agent scale, fp16 split into the padded in0 planes
            const long long t_conv0 = tacc ? clock64() : 0;
            if (et < FM_NL * FM_A) (&ms->amax[0][0])[et] = 0;
            if (et == 64) ms->xflag = 0;
            fm_zero(sm_base + FM_R2, 2 * fm_planes(1) * fm_lbo(1), et);       // act1 borders
            if (it == 0) {   // epilogue constants (weights: never produced by the kernel in front of this one)
                float* cs = reinterpret_cast<float*>(sm + FM_CST);
                for (int i = et; i < FM_NL * 2 * 128; i += FM_EPI_THREADS) cs[i] = __ldg(A.consts + i);
            }
            fm_wait(&ms->xraw_full, it & 1);
            const float* xs = reinterpret_cast<const float*>(sm + FM_XRAW);
            if (!bulk) {
                // ragged last tile, unaligned or host-mapped inputs: one coalesced pass of plain loads into the same buffer
                const float* xg = A.x + (size_t)tile * FM_A * 363;
                float* xw = reinterpret_cast<float*>(sm + FM_XRAW);
                for (int i = et; i < na * 363; i += FM_EPI_THREADS) xw[i] = __ldcg(xg + i);
            }
            fm_epi_sync();
            {
                // one warp per agent: scale from max |x|, then the agent's 13 x 16 padded pixels (no barrier in between)
                const int a = warp;
                float m = 0.f;
                if (a < na)
                    for (int i = lane; i < 363; i += 32) m = fmaxf(m, fabsf(xs[a * 363 + i]));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                const int e0 = fm_scale_exp(__float_as_uint(m));
                const float mul = fm_pow2(e0);
                if (lane == 0) {
                    ms->mul0[a] = mul;
                    ms->inv0[a] = fm_pow2(-e0);
                    const float bound = m * __ldg(cst + FM_CONST_MISC) + __ldg(cst + FM_CONST_MISC + 1);
                    const int e1 = fm_scale_exp(__float_as_uint(bound));
                    ms->mul1[a] = fm_pow2(e1);
                    ms->inv1[a] = fm_pow2(-e1);
                }
                uint32_t any_lo = 0;
                for (int i = lane; i < 13 * 16; i += 32) {
                    const int y = i >> 4, x = i & 15, row = y * 128 + a * 16 + x;
                    uint4 hi = make_uint4(0, 0, 0, 0), lo = make_uint4(0, 0, 0, 0);
                    if (y >= 1 && y <= 11 && x >= 1 && x <= 11 && a < na) {
                        const float* p = xs + a * 363 + (y - 1) * 11 + (x - 1);
                        const float v0 = p[0] * mul, v1 = p[121] * mul, v2 = p[242] * mul;
                        const __half2 h01 = __floats2half2_rn(v0, v1), h2 = __floats2half2_rn(v2, 0.f);
                        const float2 f01 = __half22float2(h01), f2 = __half22float2(h2);
                        const __half2 l01 = __floats2half2_rn(v0 - f01.x, v1 - f01.y), l2 = __floats2half2_rn(v2 - f2.x, 0.f);
                        // K slot of a pixel: [x0 x1 x2 | x0 x1 x2 | 0 0] -- the filter image holds W_hi in the first triple and
                        // W_lo in the second, so one MMA accumulates x_hi * (W_hi + W_lo)
                        const uint32_t w01 = *reinterpret_cast<const uint32_t*>(&h01), w2 = *reinterpret_cast<const uint32_t*>(&h2);
                        hi.x = w01; hi.y = (w2 & 0xFFFFu) | (w01 << 16); hi.z = (w01 >> 16) | (w2 << 16);
                        lo.x = *reinterpret_cast<const uint32_t*>(&l01); lo.y = *reinterpret_cast<const uint32_t*>(&l2);
                        any_lo |= (lo.x | lo.y) & 0x7FFF7FFFu;
                    }
                    fm_sts16(sm_base + FM_R1 + row * 16, hi);
                    fm_sts16(sm_base + FM_R1 + fm_lbo(0) + row * 16, lo);
                }
                if (__any_sync(0xffffffffu, any_lo != 0) && lane == 0) atomicOr(&ms->xflag, 1u);
            }
            fence_proxy_async_smem();
            fm_arrive_warp(&ms->xraw_free);
            fm_epi_sync();                     // xflag / act1 zeroes / in0 complete in every warp
            if (tacc) atomicAdd(&tacc[19], (unsigned long long)(clock64() - t_conv0));

            // ---- conv0: five pairs of image rows (M tiles 2j, 2j + 1 = image rows y = 2j, 2j + 1 of the 8 agents); this
            //      warpgroup's 64-row block = agents 4h .. 4h + 3, all 32 channels; y pairs are the two accumulators, x
            //      pairs rows l ^ 1 = lanes 4 apart
            {
                const bool has_lo = ms->xflag != 0;
                FM_T0();
                fm_wait(&ms->w_full[ring.slot], ring.phase);
                FM_ACC(6);
                const uint32_t a_hi = sm_base + FM_R1 + h * 64 * 16;
                const uint32_t bs = sm_base + FM_RING + ring.slot * FM_SLOT_BYTES;
                const float* cs = reinterpret_cast<const float*>(sm + FM_CST);
                for (int j = 0; j < 5; ++j) {
                    float acc[2][16];           // [tt]
                    if (has_lo) fm_conv0_mma<true>(acc, a_hi, bs, j);
                    else fm_conv0_mma<false>(acc, a_hi, bs, j);
                    wgmma_wait<0>();
#pragma unroll
                    for (int i = 0; i < 16; i += 2) {
                        const int row = 64 * h + wg_row(wt, i), c = wg_col(wt, i);
                        const int a = row >> 4, x = row & 15;
                        const float inv = ms->inv0[a], mul = ms->mul1[a];
                        float v[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float k = cs[c + e] * inv, sh = cs[128 + c + e];
                            const float u = fmaxf(fmaxf(fmaf(acc[0][i + e], k, sh), fmaf(acc[1][i + e], k, sh)), 0.f);
                            v[e] = fmaxf(u, __shfl_xor_sync(0xffffffffu, u, 4)) * mul;
                        }
                        if ((x & 1) == 0 && x < 10 && a < na) {
                            const int orow = fm_aw(1) + a * fm_wp(1) + (x >> 1) + 1 + j * fm_aw(1);
                            const __half2 hh = __floats2half2_rn(v[0], v[1]);
                            const float2 f = __half22float2(hh);
                            const __half2 ll = __floats2half2_rn(v[0] - f.x, v[1] - f.y);
                            const uint32_t addr = sm_base + FM_R2 + (c >> 3) * fm_lbo(1) + orow * 16 + (c & 7) * 2;
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&hh)) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr + fm_planes(1) * fm_lbo(1)),
                                         "r"(*reinterpret_cast<const uint32_t*>(&ll)) : "memory");
                        }
                    }
                }
                fm_arrive_warp(&ms->w_free[ring.slot]);
                ring.advance();
                fence_proxy_async_smem();
                fm_epi_sync();
                FM_ACC(26);
            }
            fm_epilogue_dyn<1>(sm, sm_base, ms, ring, na, q, h, lane, et, tacc);
            fm_epilogue_dyn<2>(sm, sm_base, ms, ring, na, q, h, lane, et, tacc);
            fm_epilogue_dyn<3>(sm, sm_base, ms, ring, na, q, h, lane, et, tacc);
            fm_epilogue_dyn<4>(sm, sm_base, ms, ring, na, q, h, lane, et, tacc);
            // ---- compress MLP: rows 0..7 of the tile are the agents
            {
                constexpr int SROW = fm_srow(5);
                float acc[1][fm_af(5)];
                fm_mma_layer<5>(sm_base, ms, ring, h, acc, tacc);
                fm_epi_sync();
                FM_T0();
                float* sacc = reinterpret_cast<float*>(sm + fm_in_base(5));
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                    const int row = wg_row(wt, i), col = h * 64 + wg_col(wt, i);
                    if (row < FM_A) *reinterpret_cast<float2*>(sacc + row * SROW + col) = make_float2(acc[0][i], acc[0][i + 1]);
                }
                fm_epi_sync();
                if (q == 0 && lane < FM_A && lane < na) {
                    const int a = lane;
                    const float inv = fm_pow2(-fm_scale_exp(ms->amax[4][a]));
                    const float* cs = reinterpret_cast<const float*>(sm + FM_CST) + 5 * 256 + h * 64;
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        float u[16];
                        fm_block_vals(sacc + a * SROW + h * 64 + 16 * b, cs + 16 * b, inv, u);
                        float* dst = A.feat + (size_t)(tile * FM_A + a) * 128 + h * 64 + 16 * b;
#pragma unroll
                        for (int i = 0; i < 16; i += 4)
                            *reinterpret_cast<float4*>(dst + i) = make_float4(u[i], u[i + 1], u[i + 2], u[i + 3]);
                    }
                }
                fm_epi_sync();      // every warp is done with this tile's shared state before the next tile resets it
                FM_ACC(31);
            }
            if (tacc) atomicAdd(&tacc[18], 1ull);
        }
    }
}

// =====================================================================================================================
// Weight preparation: per-layer power-of-two scale from max|w|, fp16 (hi, lo) images in chunk order, epilogue constants
// =====================================================================================================================
__global__ void fm_absmax_kernel(const float* __restrict__ w, int n, unsigned int* __restrict__ out) {
    float m = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

__device__ __forceinline__ __half fm_pick(float v, int islo) {
    const __half hi = __float2half_rn(v);
    return islo ? __float2half_rn(v - __half2float(hi)) : hi;
}

// one thread per fp16 element of layer L's image
__global__ void fm_prep_image_kernel(const float* __restrict__ w, __half* __restrict__ img, int L,
                                     const unsigned int* __restrict__ amax) {
    const int N = fm_n(L), idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= fm_img_bytes(L) / 2) return;
    const float mul = fm_pow2(fm_scale_exp(amax[L]));
    const int e = idx & 7;
    float v = 0.f;
    int islo = 0;
    if (L == 0) {
        // [kx][pr][plane][n (32)][8]: halves 0-2 = W_hi of input channel e, 3-5 = W_lo of channel e-3
        int r = idx >> 3;
        const int n = r & 31; r >>= 5;
        const int p = r & 1; r >>= 1;
        const int pr = r & 1, kx = r >> 1;
        const int ky = 2 * pr + p;
        islo = e >= 3;
        if (ky < 3 && e < 6) v = w[(n * 3 + (e % 3)) * 9 + ky * 3 + kx];
    } else {
        // [unit][plane][g][hi | lo][n (NC)][8]: one group g = the NC channels of a warpgroup (fm_nc), W_hi rows then W_lo
        // rows, so that A_hi x [W_hi | W_lo] is one MMA of width 2 NC.  Row split layers: one group of all N channels.
        const int Cin = fm_planes(L) * 8, KS = fm_ks(L), NC = fm_nc(L);
        int r = idx >> 3;
        const int nl = r % NC; r /= NC;
        islo = r & 1; r >>= 1;
        const int G = N / NC, g = r % G; r /= G;
        const int p = r & 1, u = r >> 1;
        const int tap = u / KS, k16 = u - tap * KS, ci = k16 * 16 + p * 8 + e, n = g * NC + nl;
        v = (L == 5) ? w[(size_t)n * 128 + ci] : w[((size_t)n * Cin + ci) * 9 + tap];
    }
    img[idx] = fm_pick(v * mul, islo);
}

// epilogue constants: [L][0][c] = BatchNorm scale / 2^ew_L, [L][1][c] = shift; misc[0] = max_c |sc_c| * sum|w_c| of conv0,
// misc[1] = max_c |sh_c| of conv0 (bound of conv0's output for inputs of magnitude <= 1)
__global__ void fm_prep_consts_kernel(const float* const* sc, const float* const* sh, const float* b5, const float* w0,
                                      const unsigned int* __restrict__ amax, float* __restrict__ cst) {
    const int c = threadIdx.x;      // 128 threads
    for (int L = 0; L < FM_NL; ++L) {
        const float inv = fm_pow2(-fm_scale_exp(amax[L]));
        float s = 0.f, t = 0.f;
        if (c < fm_n(L)) {
            s = (L < 5 ? sc[L][c] : 1.f) * inv;
            t = L < 5 ? sh[L][c] : b5[c];
        }
        cst[(L * 2) * 128 + c] = s;
        cst[(L * 2 + 1) * 128 + c] = t;
    }
    __shared__ float red[2][128];
    float b0 = 0.f, b1 = 0.f;
    if (c < 32) {
        float sw = 0.f;
        for (int i = 0; i < 27; ++i) sw += fabsf(w0[c * 27 + i]);
        b0 = fabsf(sc[0][c]) * sw;
        b1 = fabsf(sh[0][c]);
    }
    red[0][c] = b0; red[1][c] = b1;
    __syncthreads();
    if (c == 0) {
        float m0 = 0.f, m1 = 0.f;
        for (int i = 0; i < 32; ++i) { m0 = fmaxf(m0, red[0][i]); m1 = fmaxf(m1, red[1][i]); }
        cst[FM_CONST_MISC] = m0;
        cst[FM_CONST_MISC + 1] = m1;
    }
}

size_t feature_mma_arena_floats() {
    size_t bytes = 0;
    for (int L = 0; L < FM_NL; ++L) bytes += fm_img_bytes(L);
    return bytes / 4 + FM_CONST_FLOATS + 64 /* amax + pointer table */;
}

// arena layout (floats): images L0..L5 | consts | amax[8] | pointer table (sc[5], sh[5] as 64-bit)
int launch_prep_feature_mma(const float* const* conv_w, const float* compress_w, const float* const* sc,
                            const float* const* sh, const float* b5, float* arena, cudaStream_t st) {
    size_t off = 0;
    unsigned char* base = reinterpret_cast<unsigned char*>(arena);
    size_t img_off[FM_NL];
    for (int L = 0; L < FM_NL; ++L) { img_off[L] = off; off += fm_img_bytes(L); }
    float* cst = reinterpret_cast<float*>(base + off);
    unsigned int* amax = reinterpret_cast<unsigned int*>(cst + FM_CONST_FLOATS);
    const float** ptrs = reinterpret_cast<const float**>(amax + 8);
    GPP_CUDA_OK(cudaMemsetAsync(amax, 0, 32, st));
    static const int cin[6] = {3, 32, 32, 64, 64, 128};
    for (int L = 0; L < FM_NL; ++L) {
        const float* w = L < 5 ? conv_w[L] : compress_w;
        const int n = L < 5 ? fm_n(L) * cin[L] * 9 : 128 * 128;
        fm_absmax_kernel<<<32, 256, 0, st>>>(w, n, amax + L);
        GPP_LAUNCH_CHECK();
    }
    for (int L = 0; L < FM_NL; ++L) {
        const int n = fm_img_bytes(L) / 2;
        fm_prep_image_kernel<<<(n + 255) / 256, 256, 0, st>>>(L < 5 ? conv_w[L] : compress_w,
                                                              reinterpret_cast<__half*>(base + img_off[L]), L, amax);
        GPP_LAUNCH_CHECK();
    }
    const float* host_ptrs[10];
    for (int l = 0; l < 5; ++l) { host_ptrs[l] = sc[l]; host_ptrs[5 + l] = sh[l]; }
    GPP_CUDA_OK(cudaMemcpyAsync(ptrs, host_ptrs, sizeof(host_ptrs), cudaMemcpyHostToDevice, st));
    GPP_CUDA_OK(cudaStreamSynchronize(st));          // host_ptrs is a stack array
    fm_prep_consts_kernel<<<1, 128, 0, st>>>(ptrs, ptrs + 5, b5, conv_w[0], amax, cst);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

static unsigned long long* g_fm_timing = nullptr;
int debug_feature_mma_timing(unsigned long long* out32) {
    if (!g_fm_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out32, g_fm_timing, 320, cudaMemcpyDeviceToHost);
    cudaMemset(g_fm_timing, 0, 320);
    return GPP_OK;
}

int launch_feature_mma_kernel(const FeArgs& fa, const float* arena, int x_bulk, cudaStream_t st) {
    FmArgs a;
    a.x = fa.x; a.feat = fa.feat; a.total_agents = fa.total_agents;
    a.num_tiles = (fa.total_agents + FM_A - 1) / FM_A;
    const unsigned char* base = reinterpret_cast<const unsigned char*>(arena);
    size_t off = 0;
    for (int L = 0; L < FM_NL; ++L) { a.img[L] = base + off; off += fm_img_bytes(L); }
    a.consts = reinterpret_cast<const float*>(base + off);
    a.x_bulk = (x_bulk && (reinterpret_cast<uintptr_t>(fa.x) & 15) == 0) ? 1 : 0;
    a.pdl = fa.pdl;
    a.timing = nullptr;
    if (debug_option(DBG_TC_TIMING)) {
        if (!g_fm_timing) { cudaMalloc(&g_fm_timing, 320); cudaMemset(g_fm_timing, 0, 320); }
        a.timing = g_fm_timing;
    }
    static SmemConfig smem_cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(feature_mma_kernel, smem_cfg, FM_SMEM_BYTES));
    const int grid = a.num_tiles < sm_count() ? a.num_tiles : sm_count();
    GPP_CUDA_OK(launch_maybe_pdl(feature_mma_kernel, grid, FM_THREADS, FM_SMEM_BYTES, st, fa.pdl, a));
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp
