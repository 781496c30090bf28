// Batched expert solver: conflict-based search (CBS) minimising the sum of costs, one warp per case.  It replaces the
// reference's prebuilt `ecbs` binary (onlineExpert/ECBS_onlineExpert.py, offlineExpert/CasesGenerator.py:283-340),
// whose guarantee (SoC <= 1.1 x optimal at w = 1.1) an optimal SoC meets.  Every tie is fixed by the contract in
// include/gnnpp_b200.h (gpp_expert_solve) and DESIGN.md section 3.8; oracle/solver_oracle.py restates it.
//
// Work per case varies by orders of magnitude, so the grid is persistent: each warp takes cases from an atomic counter.
// Low level: a bit-parallel BFS over time layers.  A layer is W row masks of 64 bits (bit y of row x = cell (x, y));
// lane l owns rows l and l + 32.  The current layer sits in shared memory (any lane reads a neighbour row), every
// layer also goes to the warp's global scratch for the backtrack.  Constraints are few and applied by lane 0.
// High level: node pool, binary-heap open list, constraint list and paths in per-warp global scratch.  A node stores
// only its parent, the constrained agent, the constraint and that agent's new path; a node's constraints and paths
// are rebuilt by walking its parent chain.
#include <climits>

#include "common.cuh"

namespace gpp {

constexpr int SV_MAX_N = 64, SV_MAX_W = 64, SV_MAX_H = 1024, SV_MAX_NODES = 65536;
constexpr int SV_WARPS = 4;                       // warps per block
constexpr int SV_THREADS = 32 * SV_WARPS;
constexpr size_t SV_SCRATCH_BUDGET = 2ull << 30;  // the scratch of all resident warps together, bytes
constexpr size_t SV_HEADER = 256;                 // the case counter, ahead of the per-warp scratch
enum { CON_VERTEX = 0, CON_EDGE = 1 };

struct SvNode {
    int parent, agent, soc, tau;
    int kind, t, u, v;                            // the constraint the node adds: vertex v at t, or move u -> v at t
};
struct SvCon {
    int kind, t, u, v;
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Per-warp scratch, in this order (each part 256-byte aligned):
//   layers  (H + 1) * W   u64   the BFS layers of the current low-level search
//   nodes   M             SvNode (32 B)
//   heap    M             u64   open list keys (SoC << 32 | creation index)
//   cons    M             SvCon (16 B): the constraints of the agent being replanned (a chain holds at most M - 1)
//   paths   (N + M) * (H + 1)  u16 cells x * W + y: slot a = agent a's root path, slot N + k - 1 = node k's path
struct SvLayout {
    size_t layers, nodes, heap, cons, paths, per_warp;
};
static SvLayout sv_layout(int N, int W, int H, int M) {
    SvLayout L;
    size_t o = 0;
    L.layers = o; o = align_up(o + sizeof(unsigned long long) * W * (size_t)(H + 1), 256);
    L.nodes = o;  o = align_up(o + sizeof(SvNode) * (size_t)M, 256);
    L.heap = o;   o = align_up(o + sizeof(unsigned long long) * (size_t)M, 256);
    L.cons = o;   o = align_up(o + sizeof(SvCon) * (size_t)M, 256);
    L.paths = o;  o = align_up(o + sizeof(unsigned short) * (size_t)(N + M) * (H + 1), 256);
    L.per_warp = o;
    return L;
}

struct SolveArgs {
    const unsigned char* map;   // [C][W][W]
    const int* start;           // [C][N][2]
    const int* goal;            // [C][N][2]
    int* status; int* soc; int* makespan; int* created; int* expanded; int* low_level;   // [C]
    int* tau;                   // [C][N]
    short* paths;               // [C][N][H+1]
    unsigned char* scratch;     // per-warp scratch after the header
    unsigned int* counter;
    SvLayout lay;
    int C, N, W, H, M, warps;
};

struct SvShared {
    unsigned long long rows[2][SV_MAX_W];   // current / next layer
    int start[SV_MAX_N], goal[SV_MAX_N];    // cells x * W + y
    int root_tau[SV_MAX_N];
    int cur_slot[SV_MAX_N], cur_tau[SV_MAX_N];   // the expanded node's path slot and tau per agent
    int pos0[SV_MAX_N], pos1[SV_MAX_N];     // every agent's cell at t and t + 1 (conflict search)
};

struct SvWarp {
    unsigned long long* layers;
    SvNode* nodes;
    unsigned long long* heap;
    SvCon* cons;
    unsigned short* paths;
};

// delta of action d in the backtrack order stop, up, left, down, right
__device__ __forceinline__ int sv_dx(int d) { return d == 1 ? -1 : d == 3 ? 1 : 0; }
__device__ __forceinline__ int sv_dy(int d) { return d == 2 ? -1 : d == 4 ? 1 : 0; }

__device__ __forceinline__ bool sv_has(const unsigned long long* rows, int x, int y, int W) {
    return x >= 0 && x < W && y >= 0 && y < W && ((rows[x] >> y) & 1ull);
}

// Is the move p -> c between t and t + 1 edge-constrained?  (p != c; the list holds nc constraints)
__device__ __forceinline__ bool sv_edge_banned(const SvCon* cons, int nc, int t, int p, int c) {
    for (int k = 0; k < nc; ++k) {
        const SvCon q = cons[k];
        if (q.kind == CON_EDGE && q.t == t && q.u == p && q.v == c) return true;
    }
    return false;
}

// Single-agent search under cons[0..nc).  Writes the path (tau + 1 cells) to `path` and returns tau, or -1.
// last_goal: the latest vertex constraint on the goal, or -1; tlast: the last layer any constraint acts on, or -1.
__device__ __forceinline__ int sv_low_level(SvShared& sh, const SvWarp& w, const unsigned long long freeA, const unsigned long long freeB,
                            int s, int g, int nc, int last_goal, int tlast, unsigned short* path, int W, int H) {
    const int lane = threadIdx.x & 31;
    const int rA = lane, rB = lane + 32;
    const int gx = g / W, gy = g - gx * W;
    int cur = 0;
    {
        const int sx = s / W, sy = s - sx * W;
        const unsigned long long a = rA == sx ? 1ull << sy : 0ull, b = rB == sx ? 1ull << sy : 0ull;
        if (rA < W) { sh.rows[0][rA] = a; w.layers[rA] = a; }
        if (rB < W) { sh.rows[0][rB] = b; w.layers[rB] = b; }
    }
    __syncwarp();
    int t = 0;
    for (;; ++t) {
        if (((sh.rows[cur][gx] >> gy) & 1ull) && t > last_goal) break;
        if (t == H) return -1;
        const unsigned long long* L = sh.rows[cur];
        unsigned long long* nx = sh.rows[cur ^ 1];
        unsigned long long nA = 0, nB = 0;
        if (rA < W) {
            const unsigned long long r = L[rA];
            nA = (r | (r << 1) | (r >> 1) | (rA > 0 ? L[rA - 1] : 0ull) | (rA + 1 < W ? L[rA + 1] : 0ull)) & freeA;
            nx[rA] = nA;
        }
        if (rB < W) {
            const unsigned long long r = L[rB];
            nB = (r | (r << 1) | (r >> 1) | L[rB - 1] | (rB + 1 < W ? L[rB + 1] : 0ull)) & freeB;
            nx[rB] = nB;
        }
        if (t + 1 <= tlast) {
            // the constraints on layer t + 1: vertex constraints at t + 1, edge constraints at t
            __syncwarp();
            for (int k0 = 0; k0 < nc; k0 += 32) {
                bool hit = false;
                if (k0 + lane < nc) {
                    const SvCon q = w.cons[k0 + lane];
                    hit = (q.kind == CON_VERTEX && q.t == t + 1) || (q.kind == CON_EDGE && q.t == t);
                }
                unsigned m = __ballot_sync(0xffffffffu, hit);
                if (lane == 0) {
                    while (m) {
                        const int b = __ffs(m) - 1;
                        m &= m - 1;
                        const SvCon q = w.cons[k0 + b];
                        const int vx = q.v / W, vy = q.v - vx * W;
                        if (!((nx[vx] >> vy) & 1ull)) continue;
                        bool keep = false;
                        if (q.kind == CON_EDGE) {
                            // v stays if some predecessor in L_t may still move into it
                            for (int d = 0; d < 5 && !keep; ++d) {
                                const int px = vx - sv_dx(d), py = vy - sv_dy(d);
                                if (sv_has(L, px, py, W) && !(d != 0 && sv_edge_banned(w.cons, nc, t, px * W + py, q.v)))
                                    keep = true;
                            }
                        }
                        if (!keep) nx[vx] &= ~(1ull << vy);
                    }
                }
            }
            __syncwarp();
            if (rA < W) nA = nx[rA];
            if (rB < W) nB = nx[rB];
        }
        unsigned long long* gl = w.layers + (size_t)(t + 1) * W;
        if (rA < W) gl[rA] = nA;
        if (rB < W) gl[rB] = nB;
        const bool same = (rA >= W || nA == L[rA]) && (rB >= W || nB == L[rB]);
        const bool all_same = __all_sync(0xffffffffu, same);
        __syncwarp();
        cur ^= 1;
        // no constraint acts after layer t + 1 and nothing changed: every later layer is this one
        if (tlast <= t && all_same && !((sh.rows[cur][gx] >> gy) & 1ull)) return -1;
    }
    const int tau = t;
    // backtrack: lane d < 5 tries the predecessor c - delta_d, d in the order stop, up, left, down, right
    int c = g;
    if (lane == 0) path[tau] = (unsigned short)c;
    for (int tt = tau; tt > 0; --tt) {
        bool ok = false;
        int p = -1;
        if (lane < 5) {
            const int cx = c / W, cy = c - cx * W;
            const int px = cx - sv_dx(lane), py = cy - sv_dy(lane);
            const unsigned long long* Lp = w.layers + (size_t)(tt - 1) * W;
            if (px >= 0 && px < W && py >= 0 && py < W && ((Lp[px] >> py) & 1ull)) {
                p = px * W + py;
                ok = lane == 0 || !sv_edge_banned(w.cons, nc, tt - 1, p, c);
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        c = __shfl_sync(0xffffffffu, p, __ffs(m) - 1);
        if (lane == 0) path[tt - 1] = (unsigned short)c;
    }
    __syncwarp();
    return tau;
}

// Lane 0 collects the constraints of `agent` on the chain from node `k` to the root, after `first`; the results are
// broadcast.  Returns nc.
__device__ __forceinline__ int sv_collect(const SvWarp& w, int k, int agent, SvCon first, int g, int* last_goal, int* tlast) {
    const int lane = threadIdx.x & 31;
    int nc = 0, lg = -1, tl = -1;
    if (lane == 0) {
        SvCon q = first;
        for (;;) {
            w.cons[nc++] = q;
            if (q.kind == CON_VERTEX) {
                tl = max(tl, q.t);
                if (q.v == g) lg = max(lg, q.t);
            } else {
                tl = max(tl, q.t + 1);
            }
            bool found = false;
            while (k > 0) {
                const SvNode n = w.nodes[k];
                k = n.parent;
                if (n.agent == agent) {
                    q.kind = n.kind; q.t = n.t; q.u = n.u; q.v = n.v;
                    found = true;
                    break;
                }
            }
            if (!found) break;
        }
    }
    __syncwarp();
    *last_goal = __shfl_sync(0xffffffffu, lg, 0);
    *tlast = __shfl_sync(0xffffffffu, tl, 0);
    return __shfl_sync(0xffffffffu, nc, 0);
}

__device__ __forceinline__ void sv_heap_push(unsigned long long* heap, int& n, unsigned long long key) {
    int i = n++;
    while (i > 0) {
        const int p = (i - 1) >> 1;
        if (heap[p] <= key) break;
        heap[i] = heap[p];
        i = p;
    }
    heap[i] = key;
}

__device__ __forceinline__ unsigned long long sv_heap_pop(unsigned long long* heap, int& n) {
    const unsigned long long top = heap[0], last = heap[--n];
    int i = 0;
    for (;;) {
        int c = 2 * i + 1;
        if (c >= n) break;
        if (c + 1 < n && heap[c + 1] < heap[c]) ++c;
        if (heap[c] >= last) break;
        heap[i] = heap[c];
        i = c;
    }
    if (n > 0) heap[i] = last;
    return top;
}

__device__ __forceinline__ int sv_pos(const SvShared& sh, const SvWarp& w, int a, int t, int H) {
    return t <= sh.cur_tau[a] ? (int)w.paths[(size_t)sh.cur_slot[a] * (H + 1) + t] : sh.goal[a];
}

// The first conflict of the expanded node (paths in sh.cur_slot / cur_tau).  Returns false if there is none; else
// kind, t, agents i < j and cells u (vertex: the cell; swap: i's cell at t) and v (swap: i's cell at t + 1).
__device__ __forceinline__ bool sv_first_conflict(SvShared& sh, const SvWarp& w, int N, int H, int* kind, int* ct, int* ci, int* cj,
                                  int* cu, int* cv) {
    const int lane = threadIdx.x & 31;
    int T = 0;
    for (int a = lane; a < N; a += 32) T = max(T, sh.cur_tau[a]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) T = max(T, __shfl_xor_sync(0xffffffffu, T, o));
    for (int t = 0; t <= T; ++t) {
        for (int a = lane; a < N; a += 32) {
            sh.pos0[a] = sv_pos(sh, w, a, t, H);
            sh.pos1[a] = t < T ? sv_pos(sh, w, a, t + 1, H) : -1;
        }
        __syncwarp();
        for (int pass = 0; pass < 2; ++pass) {          // 0: vertex conflicts at t, 1: swaps between t and t + 1
            if (pass == 1 && t == T) break;
            for (int half = 0; half < 2; ++half) {
                const int i = lane + 32 * half;
                int jj = INT_MAX;
                if (i < N) {
                    const int a = sh.pos0[i], b = sh.pos1[i];
                    if (pass == 0) {
                        for (int j = i + 1; j < N; ++j)
                            if (sh.pos0[j] == a) { jj = j; break; }
                    } else if (a != b) {
                        for (int j = i + 1; j < N; ++j)
                            if (sh.pos0[j] == b && sh.pos1[j] == a) { jj = j; break; }
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, jj != INT_MAX);
                if (m) {
                    const int src = __ffs(m) - 1;
                    *kind = pass == 0 ? CON_VERTEX : CON_EDGE;
                    *ct = t;
                    *ci = src + 32 * half;
                    *cj = __shfl_sync(0xffffffffu, jj, src);
                    *cu = sh.pos0[*ci];
                    *cv = sh.pos1[*ci];
                    __syncwarp();
                    return true;
                }
            }
        }
        __syncwarp();
    }
    return false;
}

__global__ void __launch_bounds__(SV_THREADS) expert_solve_kernel(const SolveArgs a) {
    __shared__ SvShared shared[SV_WARPS];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * SV_WARPS + wid;
    if (gw >= a.warps) return;
    SvShared& sh = shared[wid];
    unsigned char* base = a.scratch + (size_t)gw * a.lay.per_warp;
    SvWarp w;
    w.layers = reinterpret_cast<unsigned long long*>(base + a.lay.layers);
    w.nodes = reinterpret_cast<SvNode*>(base + a.lay.nodes);
    w.heap = reinterpret_cast<unsigned long long*>(base + a.lay.heap);
    w.cons = reinterpret_cast<SvCon*>(base + a.lay.cons);
    w.paths = reinterpret_cast<unsigned short*>(base + a.lay.paths);
    const int N = a.N, W = a.W, H = a.H, M = a.M;
    const size_t P = (size_t)H + 1;
    for (;;) {
        int c = 0;
        if (lane == 0) c = (int)atomicAdd(a.counter, 1u);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c >= a.C) break;
        // the case: free-cell rows, starts, goals
        const unsigned char* mp = a.map + (size_t)c * W * W;
        unsigned long long freeA = 0, freeB = 0;
        for (int y = 0; y < W; ++y) {
            if (lane < W && mp[(size_t)lane * W + y] == 0) freeA |= 1ull << y;
            if (lane + 32 < W && mp[(size_t)(lane + 32) * W + y] == 0) freeB |= 1ull << y;
        }
        for (int i = lane; i < N; i += 32) {
            const int* s = a.start + ((size_t)c * N + i) * 2;
            const int* g = a.goal + ((size_t)c * N + i) * 2;
            sh.start[i] = s[0] * W + s[1];
            sh.goal[i] = g[0] * W + g[1];
        }
        __syncwarp();
        int status = GPP_SOLVE_NO_SOLUTION, created = 0, expanded = 0, ll = 0, soc = 0;
        int heap_n = 0;       // meaningful in lane 0
        // root: every agent alone
        bool root_ok = true;
        for (int i = 0; i < N; ++i) {
            ++ll;
            const int tau = sv_low_level(sh, w, freeA, freeB, sh.start[i], sh.goal[i], 0, -1, -1,
                                         w.paths + (size_t)i * P, W, H);
            if (tau < 0) { root_ok = false; break; }
            if (lane == 0) sh.root_tau[i] = tau;
            soc += tau;
        }
        __syncwarp();
        if (root_ok) {
            created = 1;
            if (lane == 0) {
                SvNode r;
                r.parent = -1; r.agent = -1; r.soc = soc; r.tau = -1; r.kind = r.t = r.u = r.v = -1;
                w.nodes[0] = r;
                sv_heap_push(w.heap, heap_n, (unsigned long long)soc << 32);
            }
            __syncwarp();
            for (;;) {
                const int empty = __shfl_sync(0xffffffffu, heap_n == 0, 0);
                if (empty) { status = GPP_SOLVE_NO_SOLUTION; break; }
                unsigned long long key = 0;
                if (lane == 0) key = sv_heap_pop(w.heap, heap_n);
                key = __shfl_sync(0xffffffffu, key, 0);
                const int k = (int)(key & 0xffffffffu), ksoc = (int)(key >> 32);
                ++expanded;
                // the node's paths: the nearest replanning ancestor of every agent, else the root's
                if (lane == 0) {
                    unsigned long long seen = 0;
                    for (int i = 0; i < N; ++i) { sh.cur_slot[i] = i; sh.cur_tau[i] = sh.root_tau[i]; }
                    for (int n = k; n > 0;) {
                        const SvNode nd = w.nodes[n];
                        const unsigned long long bit = 1ull << nd.agent;
                        if (!(seen & bit)) {
                            seen |= bit;
                            sh.cur_slot[nd.agent] = N + n - 1;
                            sh.cur_tau[nd.agent] = nd.tau;
                        }
                        n = nd.parent;
                    }
                }
                __syncwarp();
                int kind, ct, ci, cj, cu, cv;
                if (!sv_first_conflict(sh, w, N, H, &kind, &ct, &ci, &cj, &cu, &cv)) {
                    status = GPP_SOLVE_SOLVED;
                    soc = ksoc;
                    break;
                }
                bool budget = false;
                for (int side = 0; side < 2 && !budget; ++side) {
                    const int agent = side == 0 ? ci : cj;
                    SvCon q;
                    q.kind = kind; q.t = ct;
                    if (kind == CON_VERTEX) { q.u = -1; q.v = cu; }
                    else if (side == 0) { q.u = cu; q.v = cv; }
                    else { q.u = cv; q.v = cu; }
                    int last_goal, tlast;
                    const int nc = sv_collect(w, k, agent, q, sh.goal[agent], &last_goal, &tlast);
                    ++ll;
                    const int tau = sv_low_level(sh, w, freeA, freeB, sh.start[agent], sh.goal[agent], nc, last_goal,
                                                 tlast, w.paths + (size_t)(N + created - 1) * P, W, H);
                    if (tau < 0) continue;
                    if (created == M) { budget = true; break; }
                    const int child_soc = ksoc - sh.cur_tau[agent] + tau;
                    if (lane == 0) {
                        SvNode nd;
                        nd.parent = k; nd.agent = agent; nd.soc = child_soc; nd.tau = tau;
                        nd.kind = q.kind; nd.t = q.t; nd.u = q.u; nd.v = q.v;
                        w.nodes[created] = nd;
                        sv_heap_push(w.heap, heap_n, ((unsigned long long)child_soc << 32) | (unsigned)created);
                    }
                    ++created;
                    __syncwarp();
                }
                if (budget) { status = GPP_SOLVE_BUDGET; break; }
            }
        }
        // outputs
        const bool solved = status == GPP_SOLVE_SOLVED;
        int mk = 0;
        for (int i = lane; i < N; i += 32) {
            a.tau[(size_t)c * N + i] = solved ? sh.cur_tau[i] : -1;
            if (solved) mk = max(mk, sh.cur_tau[i]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mk = max(mk, __shfl_xor_sync(0xffffffffu, mk, o));
        for (int i = 0; i < N; ++i) {
            short* out = a.paths + ((size_t)c * N + i) * P;
            for (int t = lane; t <= H; t += 32) out[t] = solved ? (short)sv_pos(sh, w, i, t, H) : (short)-1;
        }
        if (lane == 0) {
            a.status[c] = status;
            a.soc[c] = solved ? soc : -1;
            a.makespan[c] = solved ? mk : -1;
            a.created[c] = created;
            a.expanded[c] = expanded;
            a.low_level[c] = ll;
        }
        __syncwarp();
    }
}

// Resident warps for one call: bounded by the cases, by what the device keeps resident and by the scratch budget.
static int sv_warps(int C, const SvLayout& L) {
    int blocks_per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, expert_solve_kernel, SV_THREADS, 0) != cudaSuccess ||
        blocks_per_sm < 1)
        blocks_per_sm = 1;
    const long long resident = (long long)sm_count() * blocks_per_sm * SV_WARPS;
    const long long by_budget = (long long)(SV_SCRATCH_BUDGET / L.per_warp);
    long long w = C;
    if (resident < w) w = resident;
    if (by_budget < w) w = by_budget;
    return (int)(w < 1 ? 1 : w);
}

static bool sv_in_envelope(int N, int W, int H, int M) {
    return N >= 1 && N <= SV_MAX_N && W >= 1 && W <= SV_MAX_W && H >= 1 && H <= SV_MAX_H && M >= 1 &&
           M <= SV_MAX_NODES;
}

}  // namespace gpp

using namespace gpp;

extern "C" size_t gpp_expert_solve_workspace_bytes(int C, int N, int W, int H, int max_nodes) {
    if (C <= 0 || !sv_in_envelope(N, W, H, max_nodes)) return 0;
    const SvLayout L = sv_layout(N, W, H, max_nodes);
    return SV_HEADER + (size_t)sv_warps(C, L) * L.per_warp;
}

extern "C" int gpp_expert_solve(const unsigned char* map, const int* start, const int* goal, int H, int max_nodes,
                                int* status, int* soc, int* makespan, int* nodes_created, int* nodes_expanded,
                                int* low_level, int* tau, short* paths, void* workspace, size_t workspace_bytes, int C,
                                int N, int W, void* stream) {
    GPP_REQUIRE(C >= 0 && N >= 1 && W >= 1 && H >= 0 && max_nodes >= 1, GPP_ERR_INVALID,
                "expert_solve: bad sizes C=%d N=%d W=%d H=%d max_nodes=%d", C, N, W, H, max_nodes);
    GPP_REQUIRE(sv_in_envelope(N, W, H, max_nodes), GPP_ERR_UNSUPPORTED,
                "expert_solve: N=%d W=%d H=%d max_nodes=%d outside N 1..%d, W 1..%d, H 1..%d, max_nodes 1..%d", N, W, H,
                max_nodes, SV_MAX_N, SV_MAX_W, SV_MAX_H, SV_MAX_NODES);
    if (C == 0) return GPP_OK;
    GPP_REQUIRE(map && start && goal && status && soc && makespan && nodes_created && nodes_expanded && low_level &&
                tau && paths && workspace, GPP_ERR_INVALID, "expert_solve: null pointer");
    const SvLayout L = sv_layout(N, W, H, max_nodes);
    const int warps = sv_warps(C, L);
    GPP_REQUIRE(workspace_bytes >= SV_HEADER + (size_t)warps * L.per_warp, GPP_ERR_INVALID,
                "expert_solve: workspace of %zu bytes, %zu needed", workspace_bytes,
                SV_HEADER + (size_t)warps * L.per_warp);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    SolveArgs a;
    a.map = map; a.start = start; a.goal = goal;
    a.status = status; a.soc = soc; a.makespan = makespan; a.created = nodes_created; a.expanded = nodes_expanded;
    a.low_level = low_level; a.tau = tau; a.paths = paths;
    a.counter = reinterpret_cast<unsigned int*>(workspace);
    a.scratch = reinterpret_cast<unsigned char*>(workspace) + SV_HEADER;
    a.lay = L;
    a.C = C; a.N = N; a.W = W; a.H = H; a.M = max_nodes; a.warps = warps;
    GPP_CUDA_OK(cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), st));
    expert_solve_kernel<<<(warps + SV_WARPS - 1) / SV_WARPS, SV_THREADS, 0, st>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}
