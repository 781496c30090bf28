// Feature extractor for sm_90a: per-agent CNN (5 x conv3x3+BN+ReLU, 3 max-pools) + compress
// MLP, all B*N agents tiled up to 8 at a time onto persistent 16-warp CTAs.
//
// Replaces the N sequential per-agent ConvLayers/compressMLP calls of
// DecentralPlannerNet.forward (gnn_pathplanning/graphs/models/decentralplanner.py:284-290) in
// eval mode.  Activations never leave shared memory between layers.
//
// Mapping (fp32 FMA).  Shared memory delivers 4 B per lane per clock to the register file, the FMA
// pipes want 4 operands per lane per clock, so every float fetched from shared memory has to feed >= 4
// FMAs from registers.  conv1..conv4 and the MLP therefore give each lane a register tile of 4
// consecutive output channels x several pixels (or agents): the 8 lanes of a quarter-warp cover 32
// output channels, the 4 quarter-warps of a warp split the input channels of the same outputs and meet
// through two warp shuffles per accumulator.  Filters are read as LDS.128 (4 channels), activations as
// quarter-warp-uniform LDS.128 / LDS.64 (one address per quarter-warp costs nothing extra: 128-bit
// loads are served a quarter-warp at a time anyway).  conv0 (3 input channels, 100 pixels) keeps
// lane = output channel.
//
// The filters of conv1..conv4 and the compress MLP (615 KB per tile, L2-resident) stream through a
// 4-slot shared-memory ring: one thread issues 1-D bulk async copies (cp.async.bulk -> mbarrier
// complete_tx) three chunks ahead of the 16 warps that consume them.
#include "common.cuh"
#include "feature.cuh"

namespace gpp {

constexpr int FE_THREADS = 512;
constexpr int FE_WARPS = FE_THREADS / 32;
constexpr int AM = FE_AGENTS_PER_TILE;   // 8
constexpr int IN_PIX = 3 * 11 * 11;
// shared-memory map (floats)
constexpr int SZ_IN0 = AM * 3 * 144;     // [a][c][12][12]  zero border, 11x11 inside
constexpr int SZ_ACT12 = AM * 32 * 56;   // [a][c][7][8]    zero border, 5x5 inside, row stride 8
constexpr int CS34 = 34;                 // channel stride of the 2x2 maps: [c][4 pixels][AM agents] + 2 pad, so that
                                         // the quarter-warps (neighbouring channels) hit different banks
constexpr int OFF_IN0 = 0;
constexpr int OFF_ACT1 = OFF_IN0 + SZ_IN0;
constexpr int OFF_ACT2 = OFF_ACT1 + SZ_ACT12;
constexpr int OFF_ACT3 = OFF_ACT2 + SZ_ACT12;     // [64][CS34]
constexpr int OFF_ACT4 = OFF_ACT3 + 64 * CS34;    // [64][CS34]
constexpr int OFF_ACT5 = OFF_ACT4 + 64 * CS34;    // [128][AM]
constexpr int FE_ACT_FLOATS = OFF_ACT5 + 128 * AM;
// filter ring: every chunk is <= 18 KB of k-major filter rows (see WStream::issue)
constexpr int RING_SLOTS = 4;
constexpr int SLOT_FLOATS = 4608;
constexpr int OFF_RING = FE_ACT_FLOATS;
constexpr int OFF_BARS = OFF_RING + RING_SLOTS * SLOT_FLOATS;   // RING_SLOTS x uint64 "slot filled" barriers
constexpr int FE_SMEM_FLOATS = OFF_BARS + 2 * RING_SLOTS;
static_assert((OFF_RING % 4) == 0 && (OFF_BARS % 2) == 0 && (OFF_ACT3 % 4) == 0, "ring / barrier alignment");
constexpr size_t FE_SMEM_BYTES = sizeof(float) * FE_SMEM_FLOATS;
static_assert(FE_SMEM_BYTES <= 227 * 1024, "feature kernel shared memory");

// debug phase timer: thread 0 of block 0 adds the cycles since the previous mark to timing[i]
#define FE_MARK(i)                                                          \
    if (timed) {                                                            \
        const long long tn = clock64();                                     \
        atomicAdd(&A.timing[i], (unsigned long long)(tn - tprev));          \
        tprev = tn;                                                         \
    }

__device__ __forceinline__ float bn_relu(float v, float sc, float sh) {
    return fmaxf(fmaf(v, sc, sh), 0.f);
}
// sum over the 4 quarter-warps (lanes l, l^8, l^16, l^24); every lane ends with the total
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    return v;
}

// ---------------------------------------------------------------------------------------------------
// Filter stream of one agent tile.  Chunk sequence (k-major filters, row = ci*9 + tap, column = co):
//   conv1: 2 chunks of 16 input channels per pass over the work items     (18 KB each)
//   conv2: 4 chunks of 8 input channels per pass                          (18 KB)
//   conv3: 8 chunks of 8 input channels                                   (18 KB)
//   conv4: 16 chunks of 4 input channels                                  (18 KB)
//   MLP  : 4 chunks, 8 inputs of each quarter of the input range          (4 x 4 KB)
// Every thread tracks the (uniform) counters; thread 0 issues the copy that refills a slot right after the CTA-wide
// barrier that retires its chunk, three chunks ahead of the consumers.
// Measured (on the previous target GPU) and not kept: a cluster-multicast stream (one L2 read per 2 or 4 CTAs) and a
// 10-slot stream that parks the conv3 / conv4 / MLP filters in the dead ACT1 / ACT2 buffers while conv2 computes.
// ---------------------------------------------------------------------------------------------------
struct WStream {
    float* ring;
    uint64_t* full;
    uint32_t cons;      // chunks consumed since kernel start: slot = cons % RING_SLOTS, parity = (cons / RING_SLOTS) & 1
    uint32_t prod;      // chunks issued since kernel start
    int seq, seq_len;   // next chunk to issue / number of chunks of the current tile
    int n1, n2;         // conv1 / conv2 chunks of the current tile (2 / 4 per pass)

    __device__ __forceinline__ void init(float* sm_base) {
        ring = sm_base + OFF_RING;
        full = reinterpret_cast<uint64_t*>(sm_base + OFF_BARS);
        cons = 0; prod = 0; seq = 0; seq_len = 0; n1 = 0; n2 = 0;
        if (threadIdx.x == 0) {
            for (int i = 0; i < RING_SLOTS; ++i) mbar_init(full + i, 1);
            fence_mbar_init();
        }
        __syncthreads();
    }
    __device__ __forceinline__ void issue(const FeArgs& A) {
        if (threadIdx.x == 0) {
            const int slot = prod % RING_SLOTS;
            float* dst = ring + slot * SLOT_FLOATS;
            uint64_t* bar = full + slot;
            int i = seq;
            if (i < n1) {
                mbar_arrive_expect_tx(bar, 18432u);
                bulk_g2s(dst, A.w1t + (i & 1) * 4608, 18432u, bar);
            } else if ((i -= n1) < n2) {
                mbar_arrive_expect_tx(bar, 18432u);
                bulk_g2s(dst, A.w2t + (i & 3) * 4608, 18432u, bar);
            } else if ((i -= n2) < 8) {
                mbar_arrive_expect_tx(bar, 18432u);
                bulk_g2s(dst, A.w3t + i * 4608, 18432u, bar);
            } else if ((i -= 8) < 16) {
                mbar_arrive_expect_tx(bar, 18432u);
                bulk_g2s(dst, A.w4t + i * 4608, 18432u, bar);
            } else {
                i -= 16;
                mbar_arrive_expect_tx(bar, 16384u);
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    bulk_g2s(dst + ks * 1024, A.w5t + (ks * 32 + 8 * i) * 128, 4096u, bar);
            }
        }
        ++prod;
        ++seq;
    }
    // start of a tile: the ring is empty (every chunk of the previous tile was consumed)
    __device__ __forceinline__ void begin_tile(const FeArgs& A, int conv1_passes, int conv2_passes) {
        n1 = 2 * conv1_passes;
        n2 = 4 * conv2_passes;
        seq = 0;
        seq_len = n1 + n2 + 8 + 16 + 4;
#pragma unroll 1
        for (int i = 0; i < RING_SLOTS; ++i) issue(A);
    }
    // blocks until the next chunk has landed; returns its slot
    __device__ __forceinline__ const float* acquire() const {
        const uint32_t slot = cons % RING_SLOTS;
        mbar_wait(full + slot, (cons / RING_SLOTS) & 1u);
        return ring + slot * SLOT_FLOATS;
    }
    // all warps are done with the chunk: its slot is refilled with the chunk RING_SLOTS further on
    __device__ __forceinline__ void release(const FeArgs& A) {
        __syncthreads();
        ++cons;
        if (seq < seq_len) issue(A);
    }
};

// conv1 (32->32 on 5x5): 2 of the 8 input channels of a chunk (this quarter-warp's share), NR output rows
// starting at r0 of agent a, output channels co4..co4+3.  ws = the chunk's filters of input channel cl0 at co4.
template <int NR>
__device__ __forceinline__ void conv1_chunk(float (&acc)[2][5][4], const float* __restrict__ act1,
                                            const float* __restrict__ ws) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        float row[NR + 2][8];
#pragma unroll
        for (int iy = 0; iy < NR + 2; ++iy) {
            const float4 ra = ld_smem4(act1 + u * 56 + iy * 8), rb = ld_smem4(act1 + u * 56 + iy * 8 + 4);
            row[iy][0] = ra.x; row[iy][1] = ra.y; row[iy][2] = ra.z; row[iy][3] = ra.w;
            row[iy][4] = rb.x; row[iy][5] = rb.y; row[iy][6] = rb.z; row[iy][7] = rb.w;
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const float4 w4 = ld_smem4(ws + (u * 9 + t) * 32);
            const int ky = t / 3, kx = t % 3;
#pragma unroll
            for (int oy = 0; oy < NR; ++oy)
#pragma unroll
                for (int ox = 0; ox < 5; ++ox) {
                    const float v = row[oy + ky][ox + kx];
                    acc[oy][ox][0] = fmaf(w4.x, v, acc[oy][ox][0]);
                    acc[oy][ox][1] = fmaf(w4.y, v, acc[oy][ox][1]);
                    acc[oy][ox][2] = fmaf(w4.z, v, acc[oy][ox][2]);
                    acc[oy][ox][3] = fmaf(w4.w, v, acc[oy][ox][3]);
                }
        }
    }
}

// conv2 (32->64 on 5x5, pooled to 2x2): one input channel, conv rows 2py, 2py+1 x columns 0..3, 4 output channels
__device__ __forceinline__ void conv2_chunk(float (&acc)[2][4][4], const float* __restrict__ act2,
                                            const float* __restrict__ ws) {
    float row[4][8];
#pragma unroll
    for (int iy = 0; iy < 4; ++iy) {
        const float4 ra = ld_smem4(act2 + iy * 8), rb = ld_smem4(act2 + iy * 8 + 4);
        row[iy][0] = ra.x; row[iy][1] = ra.y; row[iy][2] = ra.z; row[iy][3] = ra.w;
        row[iy][4] = rb.x; row[iy][5] = rb.y; row[iy][6] = rb.z; row[iy][7] = rb.w;
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const float4 w4 = ld_smem4(ws + t * 64);
        const int ky = t / 3, kx = t % 3;
#pragma unroll
        for (int oy = 0; oy < 2; ++oy)
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) {
                const float v = row[oy + ky][ox + kx];
                acc[oy][ox][0] = fmaf(w4.x, v, acc[oy][ox][0]);
                acc[oy][ox][1] = fmaf(w4.y, v, acc[oy][ox][1]);
                acc[oy][ox][2] = fmaf(w4.z, v, acc[oy][ox][2]);
                acc[oy][ox][3] = fmaf(w4.w, v, acc[oy][ox][3]);
            }
    }
}

// 3x3 convolution on a 2x2 map (conv3 / conv4), one input channel, an agent pair, 4 output channels:
// acc[a][p][c] += w[tap(p, q)][c] * in[a][q] for the taps that land inside the map.  `in` = the channel's
// [4 pixels][AM agents] block at the agent pair, `ws` = the channel's 9 filter rows at co4 (row stride TSTR).
template <int TSTR>
__device__ __forceinline__ void conv2x2_ci(float (&acc)[2][4][4], const float* __restrict__ in,
                                           const float* __restrict__ ws) {
    float v[2][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 t2 = *reinterpret_cast<const float2*>(in + q * AM);
        v[0][q] = t2.x;
        v[1][q] = t2.y;
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const float4 w4 = ld_smem4(ws + t * TSTR);
        const int dy = t / 3 - 1, dx = t % 3 - 1;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int qy = (p >> 1) + dy, qx = (p & 1) + dx;
            if (qy < 0 || qy > 1 || qx < 0 || qx > 1) continue;
            const int q = qy * 2 + qx;
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                acc[a][p][0] = fmaf(w4.x, v[a][q], acc[a][p][0]);
                acc[a][p][1] = fmaf(w4.y, v[a][q], acc[a][p][1]);
                acc[a][p][2] = fmaf(w4.z, v[a][q], acc[a][p][2]);
                acc[a][p][3] = fmaf(w4.w, v[a][q], acc[a][p][3]);
            }
        }
    }
}

__global__ void __launch_bounds__(FE_THREADS, 1) feature_kernel(const FeArgs A) {
    extern __shared__ __align__(16) float sm[];
    float* in0 = sm + OFF_IN0;
    float* act1 = sm + OFF_ACT1;
    float* act2 = sm + OFF_ACT2;
    float* act3 = sm + OFF_ACT3;
    float* act4 = sm + OFF_ACT4;
    float* act5 = sm + OFF_ACT5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qw = lane >> 3, l8 = lane & 7;     // quarter-warp and lane within it

    float w0[27];
#pragma unroll
    for (int j = 0; j < 27; ++j) w0[j] = __ldg(A.w0t + j * 32 + lane);
    const float sc0 = __ldg(A.sc[0] + lane), sh0 = __ldg(A.sh[0] + lane);
    const bool timed = A.timing && blockIdx.x == 0 && threadIdx.x == 0;
    long long tprev = timed ? clock64() : 0;

    WStream wsm;
    wsm.init(sm);
    // zero borders of the 5x5 maps: written once, the layers only ever write the interiors
    {
        float4* z4 = reinterpret_cast<float4*>(sm + OFF_ACT1);
        constexpr int n4 = 2 * SZ_ACT12 / 4;
        for (int i = threadIdx.x; i < n4; i += FE_THREADS) z4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }

    for (int tile = blockIdx.x; tile < A.num_tiles; tile += gridDim.x) {
        const int a0 = tile * A.apt;
        const int na = min(A.apt, A.total_agents - a0);
        const int npair = (na + 1) >> 1;
        // warp-level work items: conv1 (agent, row pair {0-1, 2-3, 4}), conv2 (agent, pooled row, channel half)
        const int c1_items = na * 3, c2_items = na * 4;
        const int c1_passes = (c1_items + FE_WARPS - 1) / FE_WARPS, c2_passes = (c2_items + FE_WARPS - 1) / FE_WARPS;
        wsm.begin_tile(A, c1_passes, c2_passes);   // the first filter chunks land while the inputs are staged
        if (A.pdl && tile == (int)blockIdx.x) {
            griddep_wait();             // whatever produced x earlier in the stream is complete and visible
            griddep_launch_dependents();
        }

        // ---- stage the binary FOV tensors into the zero-bordered layout -------------------------------
        {
            const float* xg = A.x + (size_t)a0 * IN_PIX;
#pragma unroll 4
            for (int i = threadIdx.x; i < AM * 3 * 144; i += FE_THREADS) {
                const int a = i / 432, rem = i - a * 432;
                const int c = rem / 144, p = rem - c * 144;
                const int yy = p / 12 - 1, xx = p % 12 - 1;
                float v = 0.f;
                if (a < na && yy >= 0 && yy < 11 && xx >= 0 && xx < 11)
                    v = __ldcg(xg + a * IN_PIX + c * 121 + yy * 11 + xx);
                in0[i] = v;
            }
        }
        __syncthreads();
        FE_MARK(0)

        // ---- conv0 3->32 on 11x11 (+BN+ReLU) + maxpool2 -> 32 x 5x5 ---------------------------
        // item = (agent, pooled row): conv rows 2pr, 2pr+1, cols 0..9
        for (int item = warp; item < na * 5; item += FE_WARPS) {
            const int a = item / 5, pr = item - a * 5;
            float acc[2][10];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 10; ++j) acc[i][j] = 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
#pragma unroll
                for (int iy = 0; iy < 4; ++iy) {
                    const float* rp = in0 + (a * 3 + c) * 144 + (2 * pr + iy) * 12;
                    const float4 r0 = ld_smem4(rp), r1 = ld_smem4(rp + 4), r2 = ld_smem4(rp + 8);
                    const float row[12] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y,
                                           r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
#pragma unroll
                    for (int oy = 0; oy < 2; ++oy) {
                        const int ky = iy - oy;
                        if (ky < 0 || ky > 2) continue;
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                            for (int ox = 0; ox < 10; ++ox)
                                acc[oy][ox] = fmaf(w0[c * 9 + ky * 3 + kx], row[ox + kx], acc[oy][ox]);
                    }
                }
            }
            float* out = act1 + ((a * 32 + lane) * 7 + pr + 1) * 8 + 1;
#pragma unroll
            for (int px = 0; px < 5; ++px) {
                const float m0 = fmaxf(bn_relu(acc[0][2 * px], sc0, sh0), bn_relu(acc[0][2 * px + 1], sc0, sh0));
                const float m1 = fmaxf(bn_relu(acc[1][2 * px], sc0, sh0), bn_relu(acc[1][2 * px + 1], sc0, sh0));
                out[px] = fmaxf(m0, m1);
            }
        }
        __syncthreads();
        FE_MARK(1)

        // ---- conv1 32->32 on 5x5 (+BN+ReLU) -----------------------------------------------------------
        {
            const float4 sc4 = __ldg(reinterpret_cast<const float4*>(A.sc[1]) + l8);
            const float4 sh4 = __ldg(reinterpret_cast<const float4*>(A.sh[1]) + l8);
            const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, shv[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
            for (int pass = 0; pass < c1_passes; ++pass) {
                const int item = pass * FE_WARPS + warp;
                const bool live = item < c1_items;
                const int a = item / 3, rt = item - a * 3;
                const int r0 = rt * 2;
                float acc[2][5][4];
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < 5; ++j)
#pragma unroll
                        for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;
                for (int j = 0; j < 2; ++j) {
                    const float* ws = wsm.acquire() + (4 * qw) * 9 * 32 + l8 * 4;
                    if (live) {
                        const float* ap = act1 + ((a * 32 + j * 16 + 4 * qw) * 7 + r0) * 8;
#pragma unroll 1
                        for (int h = 0; h < 2; ++h) {      // 4 of the chunk's 16 input channels, two at a time
                            if (rt < 2) conv1_chunk<2>(acc, ap + h * 112, ws + h * 18 * 32);
                            else conv1_chunk<1>(acc, ap + h * 112, ws + h * 18 * 32);
                        }
                    }
                    wsm.release(A);
                }
                if (live) {
#pragma unroll
                    for (int oy = 0; oy < 2; ++oy)
#pragma unroll
                        for (int ox = 0; ox < 5; ++ox)
#pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                const float v = quad_sum(acc[oy][ox][c]);
                                if (((oy * 5 + ox) & 3) == qw && (oy == 0 || rt < 2))
                                    act2[((a * 32 + l8 * 4 + c) * 7 + r0 + oy + 1) * 8 + ox + 1] = bn_relu(v, scv[c], shv[c]);
                            }
                }
            }
        }
        __syncthreads();
        FE_MARK(2)

        // ---- conv2 32->64 on 5x5 (+BN+ReLU) + maxpool2 -> 64 x 2x2 ------------------------------
        for (int pass = 0; pass < c2_passes; ++pass) {
            const int item = pass * FE_WARPS + warp;
            const bool live = item < c2_items;
            const int a = item % na, r = item / na;
            const int cg = r & 1, py = r >> 1;
            const int co4 = cg * 32 + l8 * 4;
            float acc[2][4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;
            for (int j = 0; j < 4; ++j) {
                const float* ws = wsm.acquire() + (2 * qw) * 9 * 64 + co4;
                if (live) {
                    const float* ap = act2 + ((a * 32 + j * 8 + 2 * qw) * 7 + 2 * py) * 8;
#pragma unroll 1
                    for (int h = 0; h < 2; ++h) conv2_chunk(acc, ap + h * 56, ws + h * 9 * 64);
                }
                wsm.release(A);
            }
            if (live) {
                const float4 sc4 = __ldg(reinterpret_cast<const float4*>(A.sc[2] + co4));
                const float4 sh4 = __ldg(reinterpret_cast<const float4*>(A.sh[2] + co4));
                const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, shv[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int px = 0; px < 2; ++px) {
                        float m = 0.f;
#pragma unroll
                        for (int oy = 0; oy < 2; ++oy)
#pragma unroll
                            for (int ox = 0; ox < 2; ++ox)
                                m = fmaxf(m, bn_relu(quad_sum(acc[oy][2 * px + ox][c]), scv[c], shv[c]));
                        if (((c * 2 + px) & 3) == qw) act3[(co4 + c) * CS34 + (py * 2 + px) * AM + a] = m;
                    }
            }
        }
        __syncthreads();
        FE_MARK(3)

        // ---- conv3 64->64 on 2x2 (+BN+ReLU): warp = (channel half, agent pair), quarter-warps split the
        //      8 input channels of a chunk ---------------------------------------------------------------
        {
            const int cog = warp & 1, g = warp >> 1;
            const bool live = g < npair;
            const int co4 = cog * 32 + l8 * 4;
            float acc[2][4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;
            for (int j = 0; j < 8; ++j) {
                const float* ws = wsm.acquire() + (2 * qw) * 576 + co4;
                if (live) {
                    const float* ip = act3 + (j * 8 + 2 * qw) * CS34 + 2 * g;
                    conv2x2_ci<64>(acc, ip, ws);
                    conv2x2_ci<64>(acc, ip + CS34, ws + 576);
                }
                wsm.release(A);
            }
            if (live) {
                const float4 sc4 = __ldg(reinterpret_cast<const float4*>(A.sc[3] + co4));
                const float4 sh4 = __ldg(reinterpret_cast<const float4*>(A.sh[3] + co4));
                const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, shv[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
#pragma unroll
                for (int p = 0; p < 4; ++p)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const float v0 = bn_relu(quad_sum(acc[0][p][c]), scv[c], shv[c]);
                        const float v1 = bn_relu(quad_sum(acc[1][p][c]), scv[c], shv[c]);
                        if (p == qw)
                            *reinterpret_cast<float2*>(act4 + (co4 + c) * CS34 + p * AM + 2 * g) = make_float2(v0, v1);
                    }
            }
        }
        __syncthreads();
        FE_MARK(4)

        // ---- conv4 64->128 on 2x2 (+BN+ReLU) + maxpool2 -> 128: warp = (channel quarter, agent pair),
        //      quarter-warps split the 4 input channels of a chunk ------------------------------------
        {
            const int cog = warp & 3, g = warp >> 2;
            const bool live = g < npair;
            const int co4 = cog * 32 + l8 * 4;
            float acc[2][4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;
            for (int j = 0; j < 16; ++j) {
                const float* ws = wsm.acquire() + qw * 1152 + co4;
                if (live) conv2x2_ci<128>(acc, act4 + (j * 4 + qw) * CS34 + 2 * g, ws);
                wsm.release(A);
            }
            if (live) {
                const float4 sc4 = __ldg(reinterpret_cast<const float4*>(A.sc[4] + co4));
                const float4 sh4 = __ldg(reinterpret_cast<const float4*>(A.sh[4] + co4));
                const float scv[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, shv[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float m0 = 0.f, m1 = 0.f;
#pragma unroll
                    for (int p = 0; p < 4; ++p) {
                        m0 = fmaxf(m0, bn_relu(quad_sum(acc[0][p][c]), scv[c], shv[c]));
                        m1 = fmaxf(m1, bn_relu(quad_sum(acc[1][p][c]), scv[c], shv[c]));
                    }
                    if (c == qw) *reinterpret_cast<float2*>(act5 + (co4 + c) * AM + 2 * g) = make_float2(m0, m1);
                }
            }
        }
        __syncthreads();
        FE_MARK(5)

        // ---- compress MLP 128->128 + ReLU: warp = (channel quarter, agent pair), quarter-warps split the
        //      input features ----------------------------------------------------------------------------
        {
            const int cog = warp & 3, g = warp >> 2;
            const bool live = g < npair;
            const int co4 = cog * 32 + l8 * 4;
            float acc[2][4];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
            for (int j = 0; j < 4; ++j) {
                const float* ws = wsm.acquire() + qw * 1024 + co4;
                if (live) {
#pragma unroll
                    for (int jl = 0; jl < 8; ++jl) {
                        const float4 w4 = ld_smem4(ws + jl * 128);
                        const float2 v = *reinterpret_cast<const float2*>(act5 + (qw * 32 + 8 * j + jl) * AM + 2 * g);
                        acc[0][0] = fmaf(w4.x, v.x, acc[0][0]); acc[0][1] = fmaf(w4.y, v.x, acc[0][1]);
                        acc[0][2] = fmaf(w4.z, v.x, acc[0][2]); acc[0][3] = fmaf(w4.w, v.x, acc[0][3]);
                        acc[1][0] = fmaf(w4.x, v.y, acc[1][0]); acc[1][1] = fmaf(w4.y, v.y, acc[1][1]);
                        acc[1][2] = fmaf(w4.z, v.y, acc[1][2]); acc[1][3] = fmaf(w4.w, v.y, acc[1][3]);
                    }
                }
                wsm.release(A);
            }
            if (live) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(A.b5 + co4));
                float o[2][4];
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int c = 0; c < 4; ++c) o[a][c] = quad_sum(acc[a][c]);
                const int a = 2 * g + qw;
                if (qw < 2 && a < na) {
                    float4 r;
                    r.x = fmaxf((qw ? o[1][0] : o[0][0]) + b4.x, 0.f);
                    r.y = fmaxf((qw ? o[1][1] : o[0][1]) + b4.y, 0.f);
                    r.z = fmaxf((qw ? o[1][2] : o[0][2]) + b4.z, 0.f);
                    r.w = fmaxf((qw ? o[1][3] : o[0][3]) + b4.w, 0.f);
                    *reinterpret_cast<float4*>(A.feat + (size_t)(a0 + a) * 128 + co4) = r;
                }
            }
        }
        __syncthreads();
        FE_MARK(6)
    }
}

static unsigned long long* g_fe_timing = nullptr;  // GPP_FE_TIMING debug counters
int debug_feature_timing(unsigned long long* out7) {
    if (!g_fe_timing) return GPP_ERR_INVALID;
    cudaDeviceSynchronize();
    cudaMemcpy(out7, g_fe_timing, 56, cudaMemcpyDeviceToHost);
    cudaMemset(g_fe_timing, 0, 64);
    return GPP_OK;
}

int launch_feature_kernel(const FeArgs& fa_in, cudaStream_t st) {
    FeArgs fa = fa_in;
    static SmemConfig smem_cfg;
    GPP_CUDA_OK(ensure_dynamic_smem(feature_kernel, smem_cfg, FE_SMEM_BYTES));
    int apt = (fa.total_agents + sm_count() - 1) / sm_count();
    if (apt > AM) apt = AM;
    if (apt < 1) apt = 1;
    fa.apt = apt;
    fa.num_tiles = (fa.total_agents + apt - 1) / apt;
    fa.timing = nullptr;
    if (debug_option(DBG_FE_TIMING)) {
        if (!g_fe_timing) {
            GPP_CUDA_OK(cudaMalloc(&g_fe_timing, 64));
            GPP_CUDA_OK(cudaMemset(g_fe_timing, 0, 64));
        }
        fa.timing = g_fe_timing;
    }
    const int grid = fa.num_tiles < sm_count() ? fa.num_tiles : sm_count();
    GPP_CUDA_OK(launch_maybe_pdl(feature_kernel, grid, FE_THREADS, FE_SMEM_BYTES, st, fa.pdl, fa));
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

}  // namespace gpp
