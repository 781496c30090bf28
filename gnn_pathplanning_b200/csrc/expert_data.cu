// Device-resident expert dataset: what the reference's online-expert DataTransformer (onlineExpert/
// DataTransformer_local_onlineExpert.py) writes into one .mat file per case and what its training loader
// (dataloader/Dataloader_dcplocal_notTF_onlineExpert.py:142-157) slices back out, one step per sample:
//
//   obtainSchedule          :154-196  states (path, then the goal) and one-hot targets (next - state)
//   computeAdjacencyMatrix  :256-305  one communication radius per trajectory, grown by 10 % at every unconnected step
//   toSeqInputTensor        dataloader/statetransformer.py:133-187  the field-of-view tensor of every step
//
// Only the integer states of a case are kept on the device.  expert_radius_kernel walks each case once (radius and the
// validity of every move); expert_gather_kernel builds any set of (case, step) samples from the states on demand.  The
// per-agent arithmetic is rollout_inputs_kernel's (rollout_common.cuh): bit-exact with the reference by construction.
#include <climits>

#include "common.cuh"
#include "rollout_common.cuh"

namespace gpp {

struct ExRadiusArgs {
    const int* states;       // [R][N][2] the states of every case, case after case
    const int* case_offset;  // [C] row of the case's step 0
    const int* case_steps;   // [C] T = makespan + 1
    const int* goal;         // [C][N][2]
    double init_radius;
    double* radius;          // [C] out
    int* valid;              // [C] out
    int* bad;                // [C][2] out: (step, agent) of the first move that is not in the delta list, else (-1, -1)
    int C, N;
};

// One CTA per case.  computeAdjacencyMatrix (:273-289): the steps in order, one threshold carried from step to step and
// multiplied by 1.1 while the current step is not connected.  Connectivity only grows with the threshold, so every step
// is connected under the final one and its degrees are >= 1 (the reference's D^-1/2 has no zero-degree guard).
// obtainSchedule (:177-189): the action of step t is state[t+1] - state[t] (the goal after the last state); anything
// but the five deltas makes list.index raise.  The reference transforms agent after agent, so the first failure is the
// smallest agent, then the smallest step.
__global__ void __launch_bounds__(RO_MAX_N) expert_radius_kernel(const ExRadiusArgs a) {
    __shared__ unsigned long long adj[RO_MAX_N];
    __shared__ int px[RO_MAX_N], py[RO_MAX_N];
    __shared__ int is_conn, first_bad;
    const int c = blockIdx.x, tid = threadIdx.x, N = a.N, T = a.case_steps[c];
    const int* st = a.states + (size_t)a.case_offset[c] * N * 2;
    const int* goal = a.goal + (size_t)c * N * 2;
    if (tid == 0) first_bad = INT_MAX;
    double rad = a.init_radius;          // every thread carries the same sequence of products
    for (int t = 0; t < T; ++t) {
        if (tid < N) {
            const int x = st[((size_t)t * N + tid) * 2], y = st[((size_t)t * N + tid) * 2 + 1];
            px[tid] = x;
            py[tid] = y;
            const int* nxt = t + 1 < T ? st + ((size_t)(t + 1) * N + tid) * 2 : goal + 2 * tid;
            if (abs(nxt[0] - x) + abs(nxt[1] - y) > 1) atomicMin(&first_bad, tid * T + t);
        }
        __syncthreads();
        for (int guard = 0; guard < 4096; ++guard) {
            if (tid < N) adj[tid] = ro_adjacency_row(tid, N, px, py, rad);
            __syncthreads();
            if (tid == 0) is_conn = ro_connected(adj, N);
            __syncthreads();
            if (is_conn) break;
            rad = rad * 1.1;
        }
    }
    if (tid == 0) {
        a.radius[c] = rad;
        a.valid[c] = first_bad == INT_MAX;
        a.bad[2 * c] = first_bad == INT_MAX ? -1 : first_bad % T;
        a.bad[2 * c + 1] = first_bad == INT_MAX ? -1 : first_bad / T;
    }
}

struct ExGatherArgs {
    const int* states;       // [R][N][2]
    const int* case_offset;  // [C]
    const int* case_steps;   // [C]
    const int* row_case;     // [R] case of every state row
    const int* goal;         // [C][N][2]
    const unsigned char* map;   // [C][W][W]
    const double* radius;    // [C]
    const long long* rows;   // [B] samples = state rows
    float* x;                // [B][N][3][11][11] out or null
    long long* target;       // [B][N][5] out or null: one-hot action
    void* S;                 // [B][N][N] out (f32 / f64) or null
    int s_is_f64, B, N, W, R;
};

// One CTA per sample (case c, step t).  pathtransformer_RelativeCoordinate + load_train_data for one step:
// the field-of-view tensor, the one-hot target and D^-1/2 A D^-1/2 with A = (pdist < radius[c]), float64.
__global__ void __launch_bounds__(128) expert_gather_kernel(const ExGatherArgs a) {
    __shared__ unsigned long long adj[RO_MAX_N];
    __shared__ int px[RO_MAX_N], py[RO_MAX_N];
    __shared__ double dinv[RO_MAX_N];
    extern __shared__ unsigned int occ_bits[];          // ceil(W*W / 32) words
    const int b = blockIdx.x, tid = threadIdx.x, N = a.N, W = a.W;
    const long long row = a.rows[b];
    if (row < 0 || row >= a.R) return;                  // the caller checks the indices; never read out of bounds
    const int c = a.row_case[row], t = (int)(row - a.case_offset[c]), T = a.case_steps[c];
    const int* st = a.states + (size_t)row * N * 2;
    const int* goal = a.goal + (size_t)c * N * 2;
    const unsigned char* map = a.map + (size_t)c * W * W;
    for (int i = tid; i < (W * W + 31) / 32; i += blockDim.x) occ_bits[i] = 0u;
    if (tid < N) {
        px[tid] = st[2 * tid];
        py[tid] = st[2 * tid + 1];
    }
    __syncthreads();
    if (tid < N) {
        ro_mark_occupied(occ_bits, px[tid], py[tid], W);
        if (a.S) adj[tid] = ro_adjacency_row(tid, N, px, py, a.radius[c]);
        if (a.target) {
            const int* nxt = t + 1 < T ? st + (size_t)N * 2 + 2 * tid : goal + 2 * tid;
            const int dx = nxt[0] - px[tid], dy = nxt[1] - py[tid];
            // delta list (:34-38): up (-1, 0), left (0, -1), down (1, 0), right (0, 1), stop (0, 0)
            const int k = dx == -1 ? 0 : dy == -1 ? 1 : dx == 1 ? 2 : dy == 1 ? 3 : 4;
            long long* o = a.target + ((size_t)b * N + tid) * 5;
#pragma unroll
            for (int q = 0; q < 5; ++q) o[q] = q == k;
        }
    }
    __syncthreads();
    if (a.S) {
        if (tid < N) dinv[tid] = sqrt(1.0 / (double)__popcll(adj[tid]));    // np.sqrt(1. / deg) (:301)
        __syncthreads();
        for (int e = tid; e < N * N; e += blockDim.x) {
            const int i = e / N, j = e - i * N;
            const double v = (adj[i] >> j & 1ull) ? dinv[i] * dinv[j] : 0.0;       // (Deg @ A) @ Deg, A in {0, 1}
            if (a.s_is_f64) reinterpret_cast<double*>(a.S)[(size_t)b * N * N + e] = v;
            else reinterpret_cast<float*>(a.S)[(size_t)b * N * N + e] = (float)v;   // the loader's .float()
        }
    }
    if (a.x) {
        float* xo = a.x + (size_t)b * N * 3 * RO_WIN * RO_WIN;
        for (int e = tid; e < N * 3 * RO_WIN * RO_WIN; e += blockDim.x) xo[e] = ro_fov_value(e, px, py, goal, map, occ_bits, W);
    }
}

}  // namespace gpp

using namespace gpp;

extern "C" int gpp_expert_radius(const int* states, const int* case_offset, const int* case_steps, const int* goal,
                                 double init_radius, double* radius, int* valid, int* bad, int C, int N, void* stream) {
    GPP_REQUIRE(states && case_offset && case_steps && goal && radius && valid && bad, GPP_ERR_INVALID,
                "expert_radius: null pointer");
    GPP_REQUIRE(C >= 0 && N >= 1, GPP_ERR_INVALID, "expert_radius: bad sizes C=%d N=%d", C, N);
    GPP_REQUIRE(N >= 2 && N <= RO_MAX_N, GPP_ERR_UNSUPPORTED, "expert_radius: N=%d outside 2..%d agents", N, RO_MAX_N);
    if (C == 0) return GPP_OK;
    ExRadiusArgs a;
    a.states = states; a.case_offset = case_offset; a.case_steps = case_steps; a.goal = goal;
    a.init_radius = init_radius; a.radius = radius; a.valid = valid; a.bad = bad; a.C = C; a.N = N;
    expert_radius_kernel<<<C, RO_MAX_N, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

extern "C" int gpp_expert_gather(const int* states, const int* case_offset, const int* case_steps, const int* row_case,
                                 const int* goal, const unsigned char* map, const double* radius, const long long* rows,
                                 float* x, long long* target_onehot, void* S, int s_is_f64, int B, int N, int W, int R,
                                 void* stream) {
    GPP_REQUIRE(states && case_offset && case_steps && row_case && goal && map && radius && rows, GPP_ERR_INVALID,
                "expert_gather: null pointer");
    GPP_REQUIRE(B >= 0 && N >= 1 && W >= 1 && R >= 0, GPP_ERR_INVALID, "expert_gather: bad sizes B=%d N=%d W=%d R=%d",
                B, N, W, R);
    GPP_REQUIRE(N >= 2 && N <= RO_MAX_N, GPP_ERR_UNSUPPORTED, "expert_gather: N=%d outside 2..%d agents", N, RO_MAX_N);
    if (B == 0) return GPP_OK;
    const size_t smem = sizeof(unsigned int) * ((size_t)(W * W + 31) / 32);
    GPP_REQUIRE(smem <= 40 * 1024, GPP_ERR_UNSUPPORTED, "expert_gather: map %dx%d too large", W, W);
    ExGatherArgs a;
    a.states = states; a.case_offset = case_offset; a.case_steps = case_steps; a.row_case = row_case; a.goal = goal;
    a.map = map; a.radius = radius; a.rows = rows; a.x = x; a.target = target_onehot; a.S = S;
    a.s_is_f64 = s_is_f64; a.B = B; a.N = N; a.W = W; a.R = R;
    expert_gather_kernel<<<B, 128, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}
