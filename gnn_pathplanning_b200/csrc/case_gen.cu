// Expert case generation: the reference's offline case generator (offlineExpert/CasesGenerator.py: mapGen, img_fill,
// setup_cases) under a seeded contract, one warp per candidate.  The contract, every draw included, is
// gpp_case_generate's in include/gnnpp_b200.h and DESIGN.md section 3.9; oracle/case_gen_oracle.py restates it.
//
// A candidate's draws are indexed by (seed, candidate, phase, draw), never streamed, so any warp can build any
// candidate and the result does not depend on the grid.  The map is W row masks of 64 bits in shared memory (bit y of
// row x = cell (x, y)); lane l owns rows l and l + 32.
//   maze:   serial by nature (each walk step reads what the earlier ones marked), built by lane 0.
//   fill:   bit-parallel: each row's component bits are closed along the row (Kogge-Stone occluded fill), then grown
//           by one row up and down, until nothing changes.
//   agents: a warp prefix sum of the rows' free-cell counts; lane i draws agent i and finds its k-th free cell with
//           a binary search over the prefix and __fns in the row.  Shared starts and goals are found with atomicOr on
//           start and goal bitmaps.
#include "common.cuh"

namespace gpp {

constexpr int CG_MAX_N = 64, CG_MAX_W = 64;
constexpr int CG_WARPS = 8;                       // warps (candidates) per block
constexpr int CG_THREADS = 32 * CG_WARPS;
constexpr long long CG_MAX_DRAWS = 1ll << 31;     // maze draws per candidate: the block index stays a 32-bit word

struct CaseGenArgs {
    unsigned long long seed, first;
    unsigned char* map;      // [K][W][W]
    int* start;              // [K][N][2]
    int* goal;               // [K][N][2]
    int* status;             // [K]
    int K, N, W, aisles, walk;
};

struct CgShared {
    unsigned long long rows[CG_MAX_W + 1];        // the maze, then its free component; row W..64 stay 0
    unsigned long long sbits[CG_MAX_W], gbits[CG_MAX_W];   // the starts and goals drawn so far
    int pre[CG_MAX_W];                            // free cells in the rows before row x
};

// Philox4x32-10 (Salmon et al., SC'11): counter (c0, c1, c2, c3), key (k0, k1).
__device__ __forceinline__ uint4 cg_philox(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0, unsigned k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
}

__device__ __forceinline__ unsigned cg_word(const uint4& b, unsigned j) {
    return j == 0 ? b.x : j == 1 ? b.y : j == 2 ? b.z : b.w;
}

// A draw in [0, n): (u32 * n) >> 32, no rejection, so every candidate makes a fixed number of draws.
__device__ __forceinline__ int cg_bounded(unsigned u, unsigned n) {
    return (int)(((unsigned long long)u * n) >> 32);
}

// The maze (mapGen), by one lane: obstacle bits into rows[0..W).
__device__ void cg_maze(unsigned long long* rows, int W, int aisles, int walk, unsigned k0, unsigned k1, unsigned s0,
                        unsigned s1) {
    const unsigned half = (unsigned)(W >> 1);
    uint4 blk = make_uint4(0, 0, 0, 0);
    unsigned cur = 0xffffffffu, j = 0;
    auto draw = [&](unsigned n) {
        if ((j >> 2) != cur) {
            cur = j >> 2;
            blk = cg_philox(k0, k1, cur, 0u, s0, s1);
        }
        return cg_bounded(cg_word(blk, j++ & 3u), n);
    };
    for (int a = 0; a < aisles; ++a) {
        int col = 2 * draw(half);
        int row = 2 * draw(half);
        rows[row] |= 1ull << col;
        for (int s = 0; s < walk; ++s) {
            const bool L = col > 1, R = col < W - 2, U = row > 1, D = row < W - 2;
            const int n = (int)L + (int)R + (int)U + (int)D;
            if (n == 0) continue;                    // W = 2: no neighbour, no draw
            int q = draw((unsigned)(n - 1));         // the list's last entry is never picked (mapGen's randint)
            int r2 = row, c2 = col;
            if (L && q-- == 0) c2 = col - 2;
            else if (R && q-- == 0) c2 = col + 2;
            else if (U && q-- == 0) r2 = row - 2;
            else r2 = row + 2;
            if (!((rows[r2] >> c2) & 1ull)) {
                rows[r2] |= 1ull << c2;
                rows[(row + r2) >> 1] |= 1ull << ((col + c2) >> 1);
                row = r2;
                col = c2;
            }
        }
    }
}

// The bits of p reachable from g along runs of p, in both directions (g is a subset of p).
__device__ __forceinline__ unsigned long long cg_hclose(unsigned long long g, unsigned long long p) {
    unsigned long long gu = g, pu = p, gd = g, pd = p;
#pragma unroll
    for (int sh = 1; sh < 64; sh <<= 1) {
        gu |= pu & (gu << sh);
        pu &= pu << sh;
        gd |= pd & (gd >> sh);
        pd &= pd >> sh;
    }
    return gu | gd;
}

// Free cell number s (row-major) of the component: its row by binary search over the prefix, its column by __fns.
__device__ __forceinline__ void cg_cell(const CgShared& sh, int W, int s, int* x, int* y) {
    int lo = 0, hi = W - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sh.pre[mid] <= s) lo = mid;
        else hi = mid - 1;
    }
    const unsigned long long m = sh.rows[lo];
    const int j = s - sh.pre[lo];
    const unsigned w0 = (unsigned)m;
    const int p0 = __popc(w0);
    *x = lo;
    *y = j < p0 ? (int)__fns(w0, 0, j + 1) : 32 + (int)__fns((unsigned)(m >> 32), 0, j - p0 + 1);
}

__global__ void __launch_bounds__(CG_THREADS) case_gen_kernel(const CaseGenArgs a) {
    __shared__ CgShared shared[CG_WARPS];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * CG_WARPS + wid;
    if (c >= a.K) return;
    CgShared& sh = shared[wid];
    const int W = a.W, N = a.N;
    const unsigned long long k = a.first + (unsigned long long)c;
    const unsigned k0 = (unsigned)k, k1 = (unsigned)(k >> 32), s0 = (unsigned)a.seed, s1 = (unsigned)(a.seed >> 32);
    const int rA = lane, rB = lane + 32;
    sh.rows[rA] = sh.rows[rB] = 0;
    sh.sbits[rA] = sh.sbits[rB] = sh.gbits[rA] = sh.gbits[rB] = 0;
    if (lane == 0) sh.rows[CG_MAX_W] = 0;
    __syncwarp();
    if (lane == 0) cg_maze(sh.rows, W, a.aisles, a.walk, k0, k1, s0, s1);
    __syncwarp();

    // fill: the free component of (0, 0)
    const unsigned long long full = W == 64 ? ~0ull : (1ull << W) - 1ull;
    const unsigned long long fA = rA < W ? ~sh.rows[rA] & full : 0ull, fB = rB < W ? ~sh.rows[rB] & full : 0ull;
    unsigned long long cA = lane == 0 ? (fA & 1ull) : 0ull, cB = 0ull;
    __syncwarp();
    for (;;) {
        cA = cg_hclose(cA, fA);
        cB = cg_hclose(cB, fB);
        sh.rows[rA] = cA;
        sh.rows[rB] = cB;
        __syncwarp();
        const unsigned long long nA = (cA | (rA > 0 ? sh.rows[rA - 1] : 0ull) | sh.rows[rA + 1]) & fA;
        const unsigned long long nB = (cB | sh.rows[rB - 1] | sh.rows[rB + 1]) & fB;
        __syncwarp();                                 // these reads before the next round's writes
        if (__all_sync(0xffffffffu, nA == cA && nB == cB)) break;
        cA = nA;
        cB = nB;
    }
    unsigned char* mp = a.map + (size_t)c * W * W;
    for (int i = lane; i < W * W; i += 32) {
        const int x = i / W, y = i - x * W;
        mp[i] = (unsigned char)(((sh.rows[x] >> y) & 1ull) ^ 1ull);
    }

    // free cells before every row: an inclusive warp scan of rows 0..31, then of rows 32..63
    const int pA = __popcll(cA), pB = __popcll(cB);
    int iA = pA, iB = pB;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int tA = __shfl_up_sync(0xffffffffu, iA, o), tB = __shfl_up_sync(0xffffffffu, iB, o);
        if (lane >= o) { iA += tA; iB += tB; }
    }
    const int TA = __shfl_sync(0xffffffffu, iA, 31);
    const int F = TA + __shfl_sync(0xffffffffu, iB, 31);
    sh.pre[rA] = iA - pA;
    sh.pre[rB] = TA + iB - pB;
    __syncwarp();

    int status = GPP_CASE_TOO_FEW_FREE;
    bool dup = false;
    for (int i = lane; i < N; i += 32) {
        int sx = -1, sy = -1, gx = -1, gy = -1;
        if (F >= 2) {
            const uint4 b = cg_philox(k0, k1, (unsigned)(i >> 1), 1u, s0, s1);   // words 2i, 2i + 1 of phase 1
            const int s = cg_bounded((i & 1) ? b.z : b.x, (unsigned)F);
            const int gp = cg_bounded((i & 1) ? b.w : b.y, (unsigned)(F - 1));
            cg_cell(sh, W, s, &sx, &sy);
            cg_cell(sh, W, gp + (gp >= s), &gx, &gy);
            dup |= (atomicOr(&sh.sbits[sx], 1ull << sy) >> sy) & 1ull;
            dup |= (atomicOr(&sh.gbits[gx], 1ull << gy) >> gy) & 1ull;
        }
        int* st = a.start + ((size_t)c * N + i) * 2;
        int* gl = a.goal + ((size_t)c * N + i) * 2;
        st[0] = sx; st[1] = sy;
        gl[0] = gx; gl[1] = gy;
    }
    if (F >= 2) status = __any_sync(0xffffffffu, dup) ? GPP_CASE_SHARED_CELL : GPP_CASE_ACCEPTED;
    if (lane == 0) a.status[c] = status;
}

}  // namespace gpp

using namespace gpp;

extern "C" int gpp_case_generate(unsigned long long seed, unsigned long long first_candidate, int K, int N, int W,
                                 int aisles, int walk, unsigned char* map, int* start, int* goal, int* status,
                                 void* stream) {
    GPP_REQUIRE(K >= 0 && aisles >= 0 && walk >= 0, GPP_ERR_INVALID, "case_generate: bad sizes K=%d aisles=%d walk=%d",
                K, aisles, walk);
    GPP_REQUIRE(N >= 1 && N <= CG_MAX_N && W >= 2 && W <= CG_MAX_W &&
                (long long)aisles * (2 + (long long)walk) < CG_MAX_DRAWS, GPP_ERR_UNSUPPORTED,
                "case_generate: N=%d W=%d aisles=%d walk=%d outside N 1..%d, W 2..%d, aisles * (2 + walk) < 2^31", N,
                W, aisles, walk, CG_MAX_N, CG_MAX_W);
    if (K == 0) return GPP_OK;
    GPP_REQUIRE(map && start && goal && status, GPP_ERR_INVALID, "case_generate: null pointer");
    CaseGenArgs a;
    a.seed = seed; a.first = first_candidate;
    a.map = map; a.start = start; a.goal = goal; a.status = status;
    a.K = K; a.N = N; a.W = W; a.aisles = aisles; a.walk = walk;
    case_gen_kernel<<<(K + CG_WARPS - 1) / CG_WARPS, CG_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}
