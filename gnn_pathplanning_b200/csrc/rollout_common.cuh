// Per-agent arithmetic shared by the rollout inputs builder (rollout.cu) and the expert dataset (expert_data.cu): the
// communication graph (scipy pdist < r with a zero diagonal, as 64-bit adjacency masks), its connectivity and the
// field-of-view tensor of dataloader/statetransformer.py.  Integer / IEEE-double arithmetic: bit-exact with the
// reference by construction.
#pragma once

#include <cmath>

namespace gpp {

constexpr int RO_MAX_N = 64;        // agents per episode (one 64-bit adjacency mask per agent)
constexpr int RO_FOV = 9;           // statetransformer.py:11
constexpr int RO_HALF = 4;          // :12  FOV_width
constexpr int RO_WIN = 11;          // :14-15  FOV + 2 * border
constexpr int RO_CENTER = 5;        // :16,20-21

// Row i of the adjacency matrix (distances < r, zero diagonal) as a bit mask over the N agents.
__device__ __forceinline__ unsigned long long ro_adjacency_row(int i, int N, const int* px, const int* py, double r) {
    unsigned long long m = 0ull;
    for (int j = 0; j < N; ++j) {
        const int dx = px[i] - px[j], dy = py[i] - py[j];
        const double d = sqrt((double)(dx * dx + dy * dy));        // scipy pdist (euclidean, float64)
        if (j != i && d < r) m |= 1ull << j;
    }
    return m;
}

// isConnected (graphTools.py:396-423) counts zero eigenvalues of the Laplacian = connected components; the same
// predicate by breadth-first search over the adjacency masks.
__device__ __forceinline__ bool ro_connected(const unsigned long long* adj, int N) {
    unsigned long long seen = 1ull, frontier = 1ull;
    while (frontier) {
        unsigned long long nxt = 0ull;
        for (int i = 0; i < N; ++i)
            if (frontier >> i & 1ull) nxt |= adj[i];
        frontier = nxt & ~seen;
        seen |= nxt;
    }
    const unsigned long long all = N >= 64 ? ~0ull : ((1ull << N) - 1ull);
    return (seen & all) == all;
}

// Marks the agents' cells in the occupancy bitmap (ceil(W*W / 32) words, zeroed by the caller).
__device__ __forceinline__ void ro_mark_occupied(unsigned int* occ_bits, int x, int y, int W) {
    atomicOr(&occ_bits[(x * W + y) >> 5], 1u << ((x * W + y) & 31));
}

// Element e of the [N][3][11][11] field-of-view tensor (statetransformer.py:82-130): channel 0 obstacle window (outside
// the map = obstacle), channel 1 goal (inside the 9x9 view, else projected onto the rim of the 11x11 window, :47-66),
// channel 2 agents.  goal is the episode's [N][2] goals, map its [W][W] obstacle map.
__device__ __forceinline__ float ro_fov_value(int e, const int* px, const int* py, const int* goal,
                                              const unsigned char* map, const unsigned int* occ_bits, int W) {
    const int i = e / (3 * RO_WIN * RO_WIN), rem = e - i * 3 * RO_WIN * RO_WIN;
    const int ch = rem / (RO_WIN * RO_WIN), uv = rem - ch * RO_WIN * RO_WIN, u = uv / RO_WIN, v = uv - u * RO_WIN;
    const int cx = px[i], cy = py[i];
    float val = 0.f;
    if (ch != 1) {
        if (u >= 1 && u <= RO_FOV && v >= 1 && v <= RO_FOV) {
            const int gx = cx - RO_HALF + (u - 1), gy = cy - RO_HALF + (v - 1);
            const bool inside = gx >= 0 && gx < W && gy >= 0 && gy < W;
            if (ch == 0) val = inside ? (map[gx * W + gy] ? 1.f : 0.f) : 1.f;
            else val = inside && (occ_bits[(gx * W + gy) >> 5] >> ((gx * W + gy) & 31) & 1u) ? 1.f : 0.f;
        }
    } else {
        const int dx = goal[2 * i] - cx, dy = goal[2 * i + 1] - cy;
        int tx, ty;
        if (abs(dx) <= RO_HALF && abs(dy) <= RO_HALF) {
            tx = RO_CENTER + dx;
            ty = RO_CENTER + dy;
        } else if (dy != 0 && abs(dx) <= abs(dy)) {
            // bearing within [pi/4, 3pi/4] or [-3pi/4, -pi/4] (:56): |dx| <= |dy|; np.round = round half to even
            ty = RO_CENTER * ((dy > 0) - (dy < 0) + 1);
            tx = RO_CENTER + (int)rint((double)RO_CENTER * (double)dx / (double)abs(dy));
        } else {
            tx = RO_CENTER * ((dx > 0) - (dx < 0) + 1);
            ty = RO_CENTER + (int)rint((double)RO_CENTER * (double)dy / (double)abs(dx));
        }
        val = (u == tx && v == ty) ? 1.f : 0.f;
    }
    return val;
}

}  // namespace gpp
