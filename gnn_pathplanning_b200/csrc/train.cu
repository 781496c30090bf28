// Training-mode forward and backward of the whole planner for sm_90a (fp32 CUDA cores).
//
// Replaces, in train mode, DecentralPlannerNet.forward (gnn_pathplanning/graphs/models/decentralplanner.py
// :278-318) and the autograd pass behind `loss.backward()` (gnn_pathplanning/agents/decentralplannerlocal.py
// :297-314).  The reference calls ConvLayers once PER AGENT, so its BatchNorm batch statistics are taken over
// (B,H,W) of one agent's slice and the running statistics are updated N times per forward, in agent order;
// both are reproduced exactly here with all B*N agents batched (image index = b*N + n).
//
// Everything is a plain data-parallel kernel with fixed-order reductions (deterministic gradients); the graph
// filter forward/backward reuse the fused kernels of graph_filter.cu through the C ABI entry points.
#include "common.cuh"

namespace gpp {

static const int kC[6] = {3, 32, 32, 64, 64, 128};     // channels
static const int kH[5] = {11, 5, 5, 2, 2};             // conv input = output height/width of layer l
static inline bool pooled_after(int l) { return l == 0 || l == 2 || l == 4; }
static inline int pooled_hw(int l) { return kH[l] / 2; }

// ---------------------------------------------------------------------------------------
// forward kernels
// ---------------------------------------------------------------------------------------
// out[img][co][y][x] = b[co] + sum_{ci,ky,kx} in[img][ci][y+ky-1][x+kx-1] w[co][ci][ky][kx]   (3x3, pad 1)
__global__ void conv3x3_fwd_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                   const float* __restrict__ b, float* __restrict__ out, int M, int Cin, int Cout,
                                   int H) {
    const int HW = H * H;
    const long long total = (long long)M * Cout * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int pos = (int)(i % HW), co = (int)((i / HW) % Cout);
        const long long img = i / ((long long)HW * Cout);
        const int y = pos / H, x = pos - y * H;
        float acc = b[co];
        const float* ip = in + img * Cin * HW;
        const float* wp = w + (size_t)co * Cin * 9;
        for (int ci = 0; ci < Cin; ++ci) {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = y + ky - 1;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = x + kx - 1;
                    if (ix < 0 || ix >= H) continue;
                    acc = fmaf(ip[ci * HW + iy * H + ix], wp[ci * 9 + ky * 3 + kx], acc);
                }
            }
        }
        out[i] = acc;
    }
}

// block reduction of two doubles
__device__ __forceinline__ void block_reduce2(double& a, double& b) {
    __shared__ double sa[32], sb[32];
    for (int off = 16; off > 0; off >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b += __shfl_xor_sync(0xffffffffu, b, off);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) { sa[warp] = a; sb[warp] = b; }
    __syncthreads();
    if (warp == 0) {
        a = lane < nw ? sa[lane] : 0.0;
        b = lane < nw ? sb[lane] : 0.0;
        for (int off = 16; off > 0; off >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, off);
            b += __shfl_xor_sync(0xffffffffu, b, off);
        }
        if (lane == 0) { sa[0] = a; sb[0] = b; }
    }
    __syncthreads();
    a = sa[0];
    b = sb[0];
    __syncthreads();
}

// per (agent n, channel c): mean and biased variance over (b, y, x) of z[(b*N+n)][c][:]; one CTA per group
// Per-agent BatchNorm of one (agent, channel) group per block, fused: batch statistics (two passes, double accumulation) ->
// a = relu(gamma * (z - mean) * invstd + beta) for the group's own elements -> optional 2x2 max-pool of them.  (The
// statistics alone used to be one launch, apply and pool two more.)
__global__ void bn_stats_kernel(const float* __restrict__ z, float* __restrict__ mean, float* __restrict__ var,
                                float* __restrict__ invstd, int B, int N, int C, int HW, float eps,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ a,
                                float* __restrict__ pooled, int H, int Hp) {
    const int n = blockIdx.x / C, c = blockIdx.x - n * C;
    const int cnt = B * HW;
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = i / HW, p = i - b * HW;
        s += (double)z[((size_t)(b * N + n) * C + c) * HW + p];
    }
    block_reduce2(s, q);
    const double mu = s / cnt;
    double d2 = 0.0, zero = 0.0;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = i / HW, p = i - b * HW;
        const double d = (double)z[((size_t)(b * N + n) * C + c) * HW + p] - mu;
        d2 += d * d;
    }
    block_reduce2(d2, zero);
    const float v = (float)(d2 / cnt);
    const float muf = (float)mu, is = 1.0f / sqrtf(v + eps);
    if (threadIdx.x == 0) {
        mean[blockIdx.x] = muf;
        var[blockIdx.x] = v;
        invstd[blockIdx.x] = is;
    }
    if (!a) return;
    const float ga = gamma[c], be = beta[c];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = i / HW, p = i - b * HW;
        const size_t idx = ((size_t)(b * N + n) * C + c) * HW + p;
        a[idx] = fmaxf(fmaf((z[idx] - muf) * is, ga, be), 0.f);
    }
    if (pooled) {
        const int HWp = Hp * Hp;
        for (int i = threadIdx.x; i < B * HWp; i += blockDim.x) {
            const int b = i / HWp, pp = i - b * HWp, py = pp / Hp, px = pp - py * Hp;
            const float* zp = z + ((size_t)(b * N + n) * C + c) * HW + (2 * py) * H + 2 * px;
            const float v0 = fmaxf(fmaf((zp[0] - muf) * is, ga, be), 0.f), v1 = fmaxf(fmaf((zp[1] - muf) * is, ga, be), 0.f);
            const float v2 = fmaxf(fmaf((zp[H] - muf) * is, ga, be), 0.f), v3 = fmaxf(fmaf((zp[H + 1] - muf) * is, ga, be), 0.f);
            pooled[((size_t)(b * N + n) * C + c) * HWp + pp] = fmaxf(fmaxf(v0, v1), fmaxf(v2, v3));
        }
    }
}

// a = relu(gamma * (z - mean) * invstd + beta)
__global__ void bn_apply_relu_kernel(const float* __restrict__ z, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ a, long long total, int N,
                                     int C, int HW) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)((i / HW) % C);
        const int n = (int)((i / ((long long)HW * C)) % N);
        const int g = n * C + c;
        a[i] = fmaxf(fmaf((z[i] - mean[g]) * invstd[g], gamma[c], beta[c]), 0.f);
    }
}

// running <- (1-m) running + m stat_n, n = 0..N-1 in agent order (unbiased variance for running_var)
__global__ void bn_running_kernel(const float* __restrict__ mean, const float* __restrict__ var, float* rm, float* rv,
                                  int N, int C, int cnt, float momentum) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float m = rm[c], v = rv[c];
    const float unb = cnt > 1 ? (float)cnt / (float)(cnt - 1) : 1.f;
    for (int n = 0; n < N; ++n) {
        m = (1.f - momentum) * m + momentum * mean[n * C + c];
        v = (1.f - momentum) * v + momentum * (var[n * C + c] * unb);
    }
    rm[c] = m;
    rv[c] = v;
}

__global__ void maxpool2_fwd_kernel(const float* __restrict__ a, float* __restrict__ p, long long total, int H, int Hp) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int px = (int)(i % Hp), py = (int)((i / Hp) % Hp);
        const long long plane = i / (Hp * Hp);
        const float* ap = a + plane * H * H + (2 * py) * H + 2 * px;
        p[i] = fmaxf(fmaxf(ap[0], ap[1]), fmaxf(ap[H], ap[H + 1]));
    }
}

// out[r][o] = act(b[o] + sum_i in[r][i] w[o][i])
__global__ void linear_fwd_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ b,
                                  float* __restrict__ out, long long R, int I, int O, int relu) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < R * O; i += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(i % O);
        const long long r = i / O;
        float acc = b[o];
        const float* ip = in + r * I;
        const float* wp = w + (size_t)o * I;
        for (int k = 0; k < I; ++k) acc = fmaf(ip[k], wp[k], acc);
        out[i] = relu ? fmaxf(acc, 0.f) : acc;
    }
}

// The 128 -> 128 compress layer, one warp per row: lanes split the reduction (coalesced 512-byte reads of a weight row,
// 4 inputs per lane in registers), butterfly sum, lane o % 32 keeps output o.  The thread-per-output kernel above reads
// the weight matrix with a 512-byte stride between lanes: 55 us at 640 rows.
__global__ void __launch_bounds__(256) linear128_fwd_rowwarp_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                                    const float* __restrict__ b, float* __restrict__ out,
                                                                    long long R, int relu) {
    const long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const float4 xv = *reinterpret_cast<const float4*>(in + r * 128 + 4 * lane);
    for (int o0 = 0; o0 < 128; o0 += 32) {
        float keep = 0.f;
#pragma unroll 4
        for (int j = 0; j < 32; ++j) {
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (size_t)(o0 + j) * 128 + 4 * lane));
            float p = fmaf(xv.x, wv.x, fmaf(xv.y, wv.y, fmaf(xv.z, wv.z, xv.w * wv.w)));
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) p += __shfl_xor_sync(0xffffffffu, p, s);
            if (lane == j) keep = p;
        }
        const float v = keep + b[o0 + lane];
        out[r * 128 + o0 + lane] = relu ? fmaxf(v, 0.f) : v;
    }
}

// logits[n][b][a] = ba[a] + sum_f shared[(b*N+n)][f] wa[a][f]
__global__ void action_fwd_kernel(const float* __restrict__ shared, const float* __restrict__ wa,
                                  const float* __restrict__ ba, float* __restrict__ logits, int B, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N * 5) return;
    const int a = i % 5, r = i / 5, b = r / N, n = r - b * N;
    float acc = ba[a];
    for (int f = 0; f < 128; ++f) acc = fmaf(shared[(size_t)r * 128 + f], wa[a * 128 + f], acc);
    logits[((size_t)n * B + b) * 5 + a] = acc;
}

// ---------------------------------------------------------------------------------------
// backward kernels
// ---------------------------------------------------------------------------------------
// dshared[r][f] = sum_a dlogits[n][b][a] wa[a][f]
__global__ void action_bwd_input_kernel(const float* __restrict__ dlogits, const float* __restrict__ wa,
                                        float* __restrict__ dshared, int B, int N) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= (long long)B * N * 128) return;
    const int f = (int)(i % 128);
    const long long r = i / 128;
    const int b = (int)(r / N), n = (int)(r - (long long)b * N);
    const float* dl = dlogits + ((size_t)n * B + b) * 5;
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 5; ++a) acc = fmaf(dl[a], wa[a * 128 + f], acc);
    dshared[i] = acc;
}
// dwa[a][f] = sum_r dlogits[r][a] shared[r][f] ; dba[a] = sum_r dlogits[r][a]   (thread per (a,f), one extra per a)
// Two stages, both fixed-order (deterministic): partial sums over row chunks (products rounded to float and accumulated in
// double, as the single-thread-per-output version did), then the chunks in order.  The one-thread-per-(a,f) version
// walked all B*N rows serially: 102 us at 640 rows.
constexpr int kActChunks = 32;
__global__ void action_bwd_weight_partial_kernel(const float* __restrict__ dlogits, const float* __restrict__ shared,
                                                 double* __restrict__ partial, int B, int N) {
    const int f = threadIdx.x, chunk = blockIdx.x;          // 128 threads, kActChunks blocks
    const int M = B * N, per = (M + kActChunks - 1) / kActChunks;
    const int r0 = chunk * per, r1 = min(M, r0 + per);
    double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0}, accb[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int r = r0; r < r1; ++r) {                        // r = b * N + n: the order of the reference's row-major sum
        const int b = r / N, n = r - b * N;
        const float* dl = dlogits + ((size_t)n * B + b) * 5;
        const float sv = shared[(size_t)r * 128 + f];
#pragma unroll
        for (int a = 0; a < 5; ++a) {
            acc[a] += (double)(dl[a] * sv);
            accb[a] += (double)dl[a];
        }
    }
#pragma unroll
    for (int a = 0; a < 5; ++a) partial[((size_t)chunk * 6 + a) * 128 + f] = acc[a];
    if (f < 5) partial[((size_t)chunk * 6 + 5) * 128 + f] = accb[f];
}
__global__ void action_bwd_weight_reduce_kernel(const double* __restrict__ partial, float* __restrict__ dwa,
                                                float* __restrict__ dba) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;    // 6 * 128 threads: (a, f), a == 5: the bias sums
    if (i >= 6 * 128) return;
    const int a = i / 128, f = i - a * 128;
    if (a == 5 && f >= 5) return;
    double acc = 0.0;
    for (int c = 0; c < kActChunks; ++c) acc += partial[((size_t)c * 6 + a) * 128 + f];
    if (a < 5) dwa[a * 128 + f] = (float)acc;
    else dba[f] = (float)acc;
}

// g[i] *= (y[i] > 0)
__global__ void relu_mask_kernel(float* __restrict__ g, const float* __restrict__ y, long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        if (!(y[i] > 0.f)) g[i] = 0.f;
}

// din[r][i] = sum_o dout[r][o] w[o][i]
__global__ void linear_bwd_input_kernel(const float* __restrict__ dout, const float* __restrict__ w,
                                        float* __restrict__ din, long long R, int I, int O) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < R * I; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % I);
        const long long r = i / I;
        float acc = 0.f;
        for (int o = 0; o < O; ++o) acc = fmaf(dout[r * O + o], w[(size_t)o * I + k], acc);
        din[i] = acc;
    }
}
// partial[chunk][o][i] = sum_{r in chunk} dout[r][o] in[r][i] ; partial_b[chunk][o] = sum dout[r][o]
__global__ void linear_bwd_weight_kernel(const float* __restrict__ dout, const float* __restrict__ in,
                                         float* __restrict__ partial, float* __restrict__ partial_b, long long R, int I,
                                         int O, int rows_per_chunk) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const long long r0 = (long long)blockIdx.y * rows_per_chunk;
    const long long r1 = r0 + rows_per_chunk < R ? r0 + rows_per_chunk : R;
    if (i < O * I) {
        const int o = i / I, k = i - o * I;
        double acc = 0.0;
        for (long long r = r0; r < r1; ++r) acc += (double)(dout[r * O + o] * in[r * I + k]);
        partial[(size_t)blockIdx.y * O * I + i] = (float)acc;
    } else if (i < O * I + O) {
        const int o = i - O * I;
        double acc = 0.0;
        for (long long r = r0; r < r1; ++r) acc += (double)dout[r * O + o];
        partial_b[(size_t)blockIdx.y * O + o] = (float)acc;
    }
}
__global__ void reduce_chunks_kernel(const float* __restrict__ partial, float* __restrict__ out, int chunks, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += (double)partial[(size_t)c * n + i];
    out[i] = (float)s;
}

// da[plane][y][x] = dp[plane][y/2][x/2] if (y,x) is the (first) arg-max of its 2x2 window, else 0
__global__ void maxpool2_bwd_kernel(const float* __restrict__ a, const float* __restrict__ dp, float* __restrict__ da,
                                    long long total, int H, int Hp) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % H), y = (int)((i / H) % H);
        const long long plane = i / (H * H);
        const int py = y >> 1, px = x >> 1;
        float g = 0.f;
        if (py < Hp && px < Hp) {
            const float* ap = a + plane * H * H + (2 * py) * H + 2 * px;
            const float v[4] = {ap[0], ap[1], ap[H], ap[H + 1]};
            int best = 0;
#pragma unroll
            for (int k = 1; k < 4; ++k)
                if (v[k] > v[best]) best = k;
            if (best == (y & 1) * 2 + (x & 1)) g = dp[plane * Hp * Hp + py * Hp + px];
        }
        da[i] = g;
    }
}

// per (n,c): s1 = sum dy_eff, s2 = sum dy_eff * xhat, dy_eff = da * (a > 0), xhat = (z - mean) * invstd
// One (agent, channel) group per block: s1 = sum dy, s2 = sum dy * xhat (double), then -- the block owns every element of
// the group -- dz = gamma * invstd * (dy - s1/m - xhat * s2/m) in place over da (evaluated in double like the reference's
// CPU kernel: for groups with near-zero variance invstd is ~316 and dy - mean(dy) cancels almost exactly).
__global__ void bn_bwd_reduce_kernel(float* __restrict__ da, const float* __restrict__ a,
                                     const float* __restrict__ z, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, const float* __restrict__ gamma,
                                     double* __restrict__ s1, double* __restrict__ s2, int B, int N, int C, int HW) {
    const int n = blockIdx.x / C, c = blockIdx.x - n * C;
    const int cnt = B * HW;
    const float mu = mean[blockIdx.x], is = invstd[blockIdx.x];
    double t1 = 0.0, t2 = 0.0;
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = i / HW, p = i - b * HW;
        const size_t idx = ((size_t)(b * N + n) * C + c) * HW + p;
        const float dy = a[idx] > 0.f ? da[idx] : 0.f;
        t1 += (double)dy;
        t2 += (double)dy * (((double)z[idx] - (double)mu) * (double)is);
    }
    block_reduce2(t1, t2);
    if (threadIdx.x == 0) {
        s1[blockIdx.x] = t1;
        s2[blockIdx.x] = t2;
    }
    const double inv_m = 1.0 / (double)cnt, isd = (double)is, gad = (double)gamma[c];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int b = i / HW, p = i - b * HW;
        const size_t idx = ((size_t)(b * N + n) * C + c) * HW + p;
        const double dy = a[idx] > 0.f ? (double)da[idx] : 0.0;
        const double xhat = ((double)z[idx] - (double)mu) * isd;
        da[idx] = (float)(gad * isd * (dy - t1 * inv_m - xhat * t2 * inv_m));
    }
}
// dgamma[c] = sum_n s2[n][c], dbeta[c] = sum_n s1[n][c]
__global__ void bn_param_grad_kernel(const double* __restrict__ s1, const double* __restrict__ s2, float* dgamma,
                                     float* dbeta, int N, int C) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double g = 0.0, b = 0.0;
    for (int n = 0; n < N; ++n) {
        g += s2[n * C + c];
        b += s1[n * C + c];
    }
    dgamma[c] = (float)g;
    dbeta[c] = (float)b;
}
// dz = gamma * invstd * (dy_eff - s1/m - xhat * s2/m)     (written in place over da)
__global__ void bn_bwd_apply_kernel(float* __restrict__ da, const float* __restrict__ a, const float* __restrict__ z,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ gamma, const double* __restrict__ s1,
                                    const double* __restrict__ s2, long long total, int B, int N, int C, int HW) {
    // evaluated in double like the reference's CPU kernel (its accumulate type for float is double): for
    // (agent, channel) groups with near-zero variance invstd is ~316 and dy - mean(dy) cancels almost exactly
    const double inv_m = 1.0 / (double)(B * HW);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)((i / HW) % C);
        const int n = (int)((i / ((long long)HW * C)) % N);
        const int g = n * C + c;
        const double dy = a[i] > 0.f ? (double)da[i] : 0.0;
        const double is = (double)invstd[g];
        const double xhat = ((double)z[i] - (double)mean[g]) * is;
        da[i] = (float)((double)gamma[c] * is * (dy - s1[g] * inv_m - xhat * s2[g] * inv_m));
    }
}

// din[img][ci][y][x] = sum_{co,ky,kx} dz[img][co][y+1-ky][x+1-kx] w[co][ci][ky][kx]
__global__ void conv3x3_bwd_input_kernel(const float* __restrict__ dz, const float* __restrict__ w,
                                         float* __restrict__ din, int M, int Cin, int Cout, int H) {
    const int HW = H * H;
    const long long total = (long long)M * Cin * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int pos = (int)(i % HW), ci = (int)((i / HW) % Cin);
        const long long img = i / ((long long)HW * Cin);
        const int y = pos / H, x = pos - y * H;
        float acc = 0.f;
        const float* dp = dz + img * Cout * HW;
        for (int co = 0; co < Cout; ++co) {
            const float* wp = w + ((size_t)co * Cin + ci) * 9;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int oy = y + 1 - ky;
                if (oy < 0 || oy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int ox = x + 1 - kx;
                    if (ox < 0 || ox >= H) continue;
                    acc = fmaf(dp[co * HW + oy * H + ox], wp[ky * 3 + kx], acc);
                }
            }
        }
        din[i] = acc;
    }
}
// partial[chunk][co][ci][tap] = sum_{img in chunk, pos} dz[img][co][pos] in[img][ci][pos + tap - 1]
// partial_b[chunk][co] = sum dz[img][co][pos]                                  (one extra thread per co)
__global__ void conv3x3_bwd_weight_kernel(const float* __restrict__ dz, const float* __restrict__ in,
                                          float* __restrict__ partial, float* __restrict__ partial_b, int M, int Cin,
                                          int Cout, int H, int imgs_per_chunk) {
    const int HW = H * H;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int m0 = blockIdx.y * imgs_per_chunk;
    const int m1 = min(M, m0 + imgs_per_chunk);
    const int nW = Cout * Cin * 9;
    if (i < nW) {
        const int tap = i % 9, ci = (i / 9) % Cin, co = i / (9 * Cin);
        const int ky = tap / 3, kx = tap - ky * 3;
        // weight gradients are long sums with heavy cancellation: per-image fp32 dot products, fp64 across images
        double acc = 0.0;
        for (int img = m0; img < m1; ++img) {
            const float* dp = dz + ((size_t)img * Cout + co) * HW;
            const float* ip = in + ((size_t)img * Cin + ci) * HW;
            float t = 0.f;
            for (int y = 0; y < H; ++y) {
                const int iy = y + ky - 1;
                if (iy < 0 || iy >= H) continue;
                for (int x = 0; x < H; ++x) {
                    const int ix = x + kx - 1;
                    if (ix < 0 || ix >= H) continue;
                    t = fmaf(dp[y * H + x], ip[iy * H + ix], t);
                }
            }
            acc += (double)t;
        }
        partial[(size_t)blockIdx.y * nW + i] = (float)acc;
    } else if (i < nW + Cout) {
        const int co = i - nW;
        double acc = 0.0;
        for (int img = m0; img < m1; ++img) {
            const float* dp = dz + ((size_t)img * Cout + co) * HW;
            for (int p = 0; p < HW; ++p) acc += (double)dp[p];
        }
        partial_b[(size_t)blockIdx.y * Cout + co] = (float)acc;
    }
}

// ---------------------------------------------------------------------------------------
// Row-tiled convolution kernels (H = 11, 5, 2 known at compile time).  A thread owns one output row (forward,
// input gradient) or the 9 taps of one (co, ci) filter (weight gradient), keeps it in registers and reads whole
// rows of its operands, so every loaded float feeds 3 (rows) to 4.5 (taps) FMAs instead of 0.5.  The order
// of the fp32 additions into every output is exactly that of the one-output-per-thread kernels above
// (ci/co outer, ky, kx; taps outside the map contribute fma(0, w, acc) = acc), so results are bit-identical.
// ---------------------------------------------------------------------------------------
template <int H>
__global__ void __launch_bounds__(256) conv3x3_fwd_rows_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                               const float* __restrict__ b, float* __restrict__ out,
                                                               int M, int Cin, int Cout) {
    constexpr int HW = H * H;
    const long long total = (long long)M * Cout * H;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i % H), co = (int)((i / H) % Cout);
        const long long img = i / ((long long)H * Cout);
        float acc[H];
        const float bias = b[co];
#pragma unroll
        for (int x = 0; x < H; ++x) acc[x] = bias;
        const float* ip = in + img * Cin * HW;
        const float* wp = w + (size_t)co * Cin * 9;
        for (int ci = 0; ci < Cin; ++ci) {
            float wv[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) wv[t] = wp[ci * 9 + t];
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = y + ky - 1;
                if (iy < 0 || iy >= H) continue;
                float r[H + 2];
                r[0] = 0.f;
                r[H + 1] = 0.f;
#pragma unroll
                for (int x = 0; x < H; ++x) r[x + 1] = ip[ci * HW + iy * H + x];
#pragma unroll
                for (int x = 0; x < H; ++x) {
                    float a = acc[x];
                    if (x > 0) a = fmaf(r[x], wv[ky * 3], a);            // the skipped taps are the ones outside the map
                    a = fmaf(r[x + 1], wv[ky * 3 + 1], a);
                    if (x < H - 1) a = fmaf(r[x + 2], wv[ky * 3 + 2], a);
                    acc[x] = a;
                }
            }
        }
        float* op = out + (img * Cout + co) * HW + y * H;
#pragma unroll
        for (int x = 0; x < H; ++x) op[x] = acc[x];
    }
}

template <int H>
__global__ void __launch_bounds__(256) conv3x3_bwd_input_rows_kernel(const float* __restrict__ dz, const float* __restrict__ w,
                                                                     float* __restrict__ din, int M, int Cin, int Cout) {
    constexpr int HW = H * H;
    const long long total = (long long)M * Cin * H;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i % H), ci = (int)((i / H) % Cin);
        const long long img = i / ((long long)H * Cin);
        float acc[H];
#pragma unroll
        for (int x = 0; x < H; ++x) acc[x] = 0.f;
        const float* dp = dz + img * Cout * HW;
        for (int co = 0; co < Cout; ++co) {
            const float* wp = w + ((size_t)co * Cin + ci) * 9;
            float wv[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) wv[t] = wp[t];
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int oy = y + 1 - ky;
                if (oy < 0 || oy >= H) continue;
                float r[H + 2];
                r[0] = 0.f;
                r[H + 1] = 0.f;
#pragma unroll
                for (int x = 0; x < H; ++x) r[x + 1] = dp[co * HW + oy * H + x];
#pragma unroll
                for (int x = 0; x < H; ++x) {           // kx = 0, 1, 2 reads output column x + 1, x, x - 1
                    float a = acc[x];
                    if (x < H - 1) a = fmaf(r[x + 2], wv[ky * 3], a);
                    a = fmaf(r[x + 1], wv[ky * 3 + 1], a);
                    if (x > 0) a = fmaf(r[x], wv[ky * 3 + 2], a);
                    acc[x] = a;
                }
            }
        }
        float* op = din + (img * Cin + ci) * HW + y * H;
#pragma unroll
        for (int x = 0; x < H; ++x) op[x] = acc[x];
    }
}

// 2x2 maps (conv3 / conv4): a row is only 2 pixels, so a thread owns the whole map of 4 consecutive images for one
// output (forward) or input (input gradient) channel: 9 filter values + 4 float4 maps feed 64 FMAs.  Same order of
// additions per output as above (channel outer, ky, kx, taps outside the map skipped).
__global__ void __launch_bounds__(256) conv3x3_fwd_2x2_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                              const float* __restrict__ b, float* __restrict__ out,
                                                              int M, int Cin, int Cout) {
    const long long total = (long long)((M + 3) / 4) * Cout;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(i % Cout);
        const int img0 = (int)(i / Cout) * 4;
        const int nimg = min(4, M - img0);
        float acc[4][4];
        const float bias = b[co];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[j][p] = bias;
        const float* wp = w + (size_t)co * Cin * 9;
        for (int ci = 0; ci < Cin; ++ci) {
            float wv[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) wv[t] = wp[ci * 9 + t];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j >= nimg) break;
                const float4 v4 = *reinterpret_cast<const float4*>(in + ((size_t)(img0 + j) * Cin + ci) * 4);
                const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int y = 0; y < 2; ++y)
#pragma unroll
                    for (int x = 0; x < 2; ++x) {
                        float a = acc[j][y * 2 + x];
#pragma unroll
                        for (int ky = 0; ky < 3; ++ky) {
                            const int iy = y + ky - 1;
                            if (iy < 0 || iy > 1) continue;
#pragma unroll
                            for (int kx = 0; kx < 3; ++kx) {
                                const int ix = x + kx - 1;
                                if (ix < 0 || ix > 1) continue;
                                a = fmaf(v[iy * 2 + ix], wv[ky * 3 + kx], a);
                            }
                        }
                        acc[j][y * 2 + x] = a;
                    }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (j >= nimg) break;
            *reinterpret_cast<float4*>(out + ((size_t)(img0 + j) * Cout + co) * 4) =
                make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
        }
    }
}

__global__ void __launch_bounds__(256) conv3x3_bwd_input_2x2_kernel(const float* __restrict__ dz, const float* __restrict__ w,
                                                                    float* __restrict__ din, int M, int Cin, int Cout) {
    const long long total = (long long)((M + 3) / 4) * Cin;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % Cin);
        const int img0 = (int)(i / Cin) * 4;
        const int nimg = min(4, M - img0);
        float acc[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[j][p] = 0.f;
        for (int co = 0; co < Cout; ++co) {
            const float* wp = w + ((size_t)co * Cin + ci) * 9;
            float wv[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) wv[t] = wp[t];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j >= nimg) break;
                const float4 v4 = *reinterpret_cast<const float4*>(dz + ((size_t)(img0 + j) * Cout + co) * 4);
                const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int y = 0; y < 2; ++y)
#pragma unroll
                    for (int x = 0; x < 2; ++x) {
                        float a = acc[j][y * 2 + x];
#pragma unroll
                        for (int ky = 0; ky < 3; ++ky) {
                            const int oy = y + 1 - ky;
                            if (oy < 0 || oy > 1) continue;
#pragma unroll
                            for (int kx = 0; kx < 3; ++kx) {
                                const int ox = x + 1 - kx;
                                if (ox < 0 || ox > 1) continue;
                                a = fmaf(v[oy * 2 + ox], wv[ky * 3 + kx], a);
                            }
                        }
                        acc[j][y * 2 + x] = a;
                    }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (j >= nimg) break;
            *reinterpret_cast<float4*>(din + ((size_t)(img0 + j) * Cin + ci) * 4) =
                make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
        }
    }
}

// thread = (co, ci): all 9 taps over the images of chunk blockIdx.y; threads past Cout*Cin: bias sums
template <int H>
__global__ void __launch_bounds__(128) conv3x3_bwd_weight_taps_kernel(const float* __restrict__ dz, const float* __restrict__ in,
                                                                      float* __restrict__ partial,
                                                                      float* __restrict__ partial_b, int M, int Cin,
                                                                      int Cout, int imgs_per_chunk) {
    constexpr int HW = H * H;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int m0 = blockIdx.y * imgs_per_chunk;
    const int m1 = min(M, m0 + imgs_per_chunk);
    const int nP = Cout * Cin;
    if (i < nP) {
        const int ci = i % Cin, co = i / Cin;
        double acc[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) acc[t] = 0.0;
        for (int img = m0; img < m1; ++img) {
            const float* dp = dz + ((size_t)img * Cout + co) * HW;
            const float* ip = in + ((size_t)img * Cin + ci) * HW;
            float tsum[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) tsum[t] = 0.f;
#pragma unroll
            for (int y = 0; y < H; ++y) {
                float d[H];
#pragma unroll
                for (int x = 0; x < H; ++x) d[x] = dp[y * H + x];
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    const int iy = y + ky - 1;
                    if (iy < 0 || iy >= H) continue;         // compile-time after unrolling
                    float r[H];
#pragma unroll
                    for (int x = 0; x < H; ++x) r[x] = ip[iy * H + x];
#pragma unroll
                    for (int x = 0; x < H; ++x) {
                        if (x > 0) tsum[ky * 3] = fmaf(d[x], r[x - 1], tsum[ky * 3]);
                        tsum[ky * 3 + 1] = fmaf(d[x], r[x], tsum[ky * 3 + 1]);
                        if (x < H - 1) tsum[ky * 3 + 2] = fmaf(d[x], r[x + 1], tsum[ky * 3 + 2]);
                    }
                }
            }
#pragma unroll
            for (int t = 0; t < 9; ++t) acc[t] += (double)tsum[t];
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) partial[(size_t)blockIdx.y * nP * 9 + (size_t)i * 9 + t] = (float)acc[t];
    } else if (i < nP + Cout) {
        const int co = i - nP;
        double acc = 0.0;
        for (int img = m0; img < m1; ++img) {
            const float* dp = dz + ((size_t)img * Cout + co) * HW;
            for (int p = 0; p < HW; ++p) acc += (double)dp[p];
        }
        partial_b[(size_t)blockIdx.y * Cout + co] = (float)acc;
    }
}

// ---------------------------------------------------------------------------------------
// workspace layout
// ---------------------------------------------------------------------------------------
struct TrainWs {
    size_t z[5], a[5], p[5], mean[5], var[5], invstd[5], s1, s2;
    size_t feat, shared, dfeat, dshared, dbuf0, dbuf1, partial, partial_b, gf_fwd, gf_bwd, total;
    int chunks;
};
static TrainWs train_layout(int B, int N, int K) {
    TrainWs L;
    const size_t M = (size_t)B * N;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off += (n + 63) / 64 * 64; return o; };
    size_t maxact = 0;
    for (int l = 0; l < 5; ++l) {
        const size_t n = M * kC[l + 1] * kH[l] * kH[l];
        L.z[l] = take(n);
        L.a[l] = take(n);
        L.p[l] = pooled_after(l) ? take(M * kC[l + 1] * pooled_hw(l) * pooled_hw(l)) : 0;
        L.mean[l] = take((size_t)N * kC[l + 1]);
        L.var[l] = take((size_t)N * kC[l + 1]);
        L.invstd[l] = take((size_t)N * kC[l + 1]);
        if (n > maxact) maxact = n;
    }
    L.s1 = take((size_t)N * 128 * 2);      // doubles
    L.s2 = take((size_t)N * 128 * 2);
    L.feat = take(M * 128);
    L.shared = take(M * 128);
    L.dfeat = take(M * 128);
    L.dshared = take(M * 128);
    L.dbuf0 = take(maxact);
    L.dbuf1 = take(maxact);
    L.chunks = (int)(M < 64 ? M : 64);
    L.partial = take((size_t)L.chunks * 128 * 64 * 9);
    L.partial_b = take((size_t)L.chunks * 128);
    L.gf_fwd = take(gpp_graph_filter_workspace_bytes(128, 128, K) / 4 + 64);
    L.gf_bwd = take(gpp_graph_filter_backward_workspace_bytes(B, N, 128, 128, K) / 4 + 64);
    L.total = off;
    return L;
}

static inline int grid_for(long long total, int block = 256) {
    long long g = (total + block - 1) / block;
    const long long cap = 148LL * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// the planner's maps are 11x11, 5x5 and 2x2: row-tiled kernels; anything else: the generic kernels
// ---------------------------------------------------------------------------------------------------------------------
// 3x3 convolution (pad 1) on 2x2 maps as a shared-memory-tiled GEMM, forward and input-gradient in one template:
//   O[img][n][p] = bias[n] + sum_k sum_q I[img][k][q] * w(n, k, tap(p, q))        p, q = the 4 pixels of the map
// FWD: n = output channel, k = input channel, tap = (qy - py + 1, qx - px + 1), w = W[n][k];
// BWD: n = input channel,  k = output channel, tap = (py - qy + 1, px - qx + 1), w = W[k][n]  (din from dz).
// Block = 16 images x 32 n (256 threads: one image x 4 n x 4 pixels per thread), K staged 8 at a time: inputs [16][8][4],
// weights [8][9][32] read from the raw [Cout][Cin][3][3] layout in contiguous runs.  The thread-per-(4 images, channel)
// kernels above read the weights with a 2.3 KB stride between lanes and launched 40-80 blocks: 96 / 73 us per call at
// 640 images; these take a few us.
// ---------------------------------------------------------------------------------------------------------------------
template <bool BWD>
__global__ void __launch_bounds__(256) conv2x2_gemm_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                           const float* __restrict__ bias, float* __restrict__ out, int M,
                                                           int K, int NO, int Cin) {
    __shared__ __align__(16) float sI[16][8][4];
    __shared__ __align__(16) float sW[8][9][32];
    const int tid = threadIdx.x, nq = tid & 7;                         // 8 n-quads = 32 n per block, 16 images,
    const int half = (tid >> 7) & 1;                                    // and the two pixel pairs {0,1} / {2,3}
    const int img_l = (tid >> 3) & 15;
    const int img0 = blockIdx.x * 16, n0 = blockIdx.y * 32;
    float acc[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float bv = (!BWD && bias) ? bias[n0 + 4 * nq + j] : 0.f;
        acc[j][0] = bv; acc[j][1] = bv;
    }
    for (int k0 = 0; k0 < K; k0 += 8) {
        __syncthreads();
        if (tid < 128) {                                                // inputs: 16 images x 8 k x float4
            const int ii = tid >> 3, kk = tid & 7;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (img0 + ii < M) v = *reinterpret_cast<const float4*>(in + ((size_t)(img0 + ii) * K + k0 + kk) * 4);
            *reinterpret_cast<float4*>(&sI[ii][kk][0]) = v;
        }
        for (int e = tid; e < 8 * 9 * 32; e += 256) {                   // weights
            int kk, t, n;
            size_t src;
            if (!BWD) {          // runs of 72 floats: w[n][k0 .. k0+7][0..8]
                n = e / 72; const int r = e - n * 72; kk = r / 9; t = r - kk * 9;
                src = ((size_t)(n0 + n) * Cin + k0 + kk) * 9 + t;
            } else {             // runs of 288 floats: w[k0+kk][n0 .. n0+31][0..8]
                kk = e / 288; const int r = e - kk * 288; n = r / 9; t = r - n * 9;
                src = ((size_t)(k0 + kk) * Cin + n0 + n) * 9 + t;
            }
            sW[kk][t][n] = w[src];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const float4 iv = *reinterpret_cast<const float4*>(&sI[img_l][kk][0]);
            const float q[4] = {iv.x, iv.y, iv.z, iv.w};
#pragma unroll
            for (int pp = 0; pp < 2; ++pp) {
                const int p = 2 * half + pp, py = p >> 1, px = p & 1;
#pragma unroll
                for (int qi = 0; qi < 4; ++qi) {
                    const int qy = qi >> 1, qx = qi & 1;
                    const int t = BWD ? ((py - qy + 1) * 3 + (px - qx + 1)) : ((qy - py + 1) * 3 + (qx - px + 1));
                    const float4 wv = *reinterpret_cast<const float4*>(&sW[kk][0][0] + ((size_t)t * 32 + 4 * nq));
                    acc[0][pp] = fmaf(q[qi], wv.x, acc[0][pp]);
                    acc[1][pp] = fmaf(q[qi], wv.y, acc[1][pp]);
                    acc[2][pp] = fmaf(q[qi], wv.z, acc[2][pp]);
                    acc[3][pp] = fmaf(q[qi], wv.w, acc[3][pp]);
                }
            }
        }
    }
    if (img0 + img_l < M) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float2*>(out + ((size_t)(img0 + img_l) * NO + n0 + 4 * nq + j) * 4 + 2 * half) =
                make_float2(acc[j][0], acc[j][1]);
    }
}

// The same formulation on 5x5 maps (conv1, conv2): block = IMGS images x 32 n, 40 threads per image = (map row, n-quad), one
// thread owns a row of 5 pixels x 4 n; K staged 8 at a time as zero-bordered 7 x 8 planes.  61 / 35 us per call before.
template <bool BWD, int IMGS>
__global__ void __launch_bounds__(40 * IMGS) conv5x5_gemm_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                           const float* __restrict__ bias, float* __restrict__ out, int M,
                                                           int K, int NO, int Cin) {
    __shared__ __align__(16) float sI[IMGS][8][7][8];       // [image][k][padded row][padded col (7 used)]
    __shared__ __align__(16) float sW[8][9][32];
    const int tid = threadIdx.x, nq = tid & 7, row = (tid >> 3) % 5, img_l = tid / 40;
    constexpr int NT = 40 * IMGS;
    const int img0 = blockIdx.x * IMGS, n0 = blockIdx.y * 32;
    for (int e = tid; e < IMGS * 8 * 7 * 8; e += NT) (&sI[0][0][0][0])[e] = 0.f;      // borders stay zero
    float acc[4][5];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float bv = (!BWD && bias) ? bias[n0 + 4 * nq + j] : 0.f;
#pragma unroll
        for (int x = 0; x < 5; ++x) acc[j][x] = bv;
    }
    for (int k0 = 0; k0 < K; k0 += 8) {
        __syncthreads();
        for (int e = tid; e < IMGS * 8 * 25; e += NT) {                   // inputs: 64 planes of 25 contiguous floats
            const int pl = e / 25, px = e - pl * 25, ii = pl >> 3, kk = pl & 7;
            float v = 0.f;
            if (img0 + ii < M) v = in[((size_t)(img0 + ii) * K + k0 + kk) * 25 + px];
            sI[ii][kk][px / 5 + 1][px % 5 + 1] = v;
        }
        for (int e = tid; e < 8 * 9 * 32; e += NT) {                   // weights (taps flipped for the input gradient)
            int kk, t, n;
            size_t src;
            if (!BWD) {
                n = e / 72; const int r = e - n * 72; kk = r / 9; t = r - kk * 9;
                src = ((size_t)(n0 + n) * Cin + k0 + kk) * 9 + t;
                sW[kk][t][n] = w[src];
            } else {
                kk = e / 288; const int r = e - kk * 288; n = r / 9; t = r - n * 9;
                src = ((size_t)(k0 + kk) * Cin + n0 + n) * 9 + t;
                sW[kk][8 - t][n] = w[src];
            }
        }
        __syncthreads();
#pragma unroll 2
        for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const float4 i0 = *reinterpret_cast<const float4*>(&sI[img_l][kk][row + ky][0]);
                const float4 i1 = *reinterpret_cast<const float4*>(&sI[img_l][kk][row + ky][4]);
                const float v[7] = {i0.x, i0.y, i0.z, i0.w, i1.x, i1.y, i1.z};
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 wv = *reinterpret_cast<const float4*>(&sW[kk][ky * 3 + kx][4 * nq]);
#pragma unroll
                    for (int x = 0; x < 5; ++x) {
                        acc[0][x] = fmaf(v[x + kx], wv.x, acc[0][x]);
                        acc[1][x] = fmaf(v[x + kx], wv.y, acc[1][x]);
                        acc[2][x] = fmaf(v[x + kx], wv.z, acc[2][x]);
                        acc[3][x] = fmaf(v[x + kx], wv.w, acc[3][x]);
                    }
                }
            }
        }
    }
    if (img0 + img_l < M) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float* dst = out + ((size_t)(img0 + img_l) * NO + n0 + 4 * nq + j) * 25 + row * 5;
#pragma unroll
            for (int x = 0; x < 5; ++x) dst[x] = acc[j][x];
        }
    }
}

static void launch_conv_fwd(const float* in, const float* w, const float* b, float* out, int M, int Cin, int Cout, int H,
                            cudaStream_t st) {
    const long long rows = (long long)M * Cout * H;
    if (H == 11) conv3x3_fwd_rows_kernel<11><<<grid_for(rows), 256, 0, st>>>(in, w, b, out, M, Cin, Cout);
    else if (H == 5 && Cin % 8 == 0 && Cout % 32 == 0)
        conv5x5_gemm_kernel<false, 4><<<dim3((M + 3) / 4, Cout / 32), 160, 0, st>>>(in, w, b, out, M, Cin, Cout, Cin);
    else if (H == 5) conv3x3_fwd_rows_kernel<5><<<grid_for(rows), 256, 0, st>>>(in, w, b, out, M, Cin, Cout);
    else if (H == 2 && Cin % 8 == 0 && Cout % 32 == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0)
        conv2x2_gemm_kernel<false><<<dim3((M + 15) / 16, Cout / 32), 256, 0, st>>>(in, w, b, out, M, Cin, Cout, Cin);
    else if (H == 2 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0)
        conv3x3_fwd_2x2_kernel<<<grid_for((long long)((M + 3) / 4) * Cout), 256, 0, st>>>(in, w, b, out, M, Cin, Cout);
    else if (H == 2) conv3x3_fwd_rows_kernel<2><<<grid_for(rows), 256, 0, st>>>(in, w, b, out, M, Cin, Cout);
    else conv3x3_fwd_kernel<<<grid_for(rows * H), 256, 0, st>>>(in, w, b, out, M, Cin, Cout, H);
}
static void launch_conv_bwd_input(const float* dz, const float* w, float* din, int M, int Cin, int Cout, int H,
                                  cudaStream_t st) {
    const long long rows = (long long)M * Cin * H;
    if (H == 11) conv3x3_bwd_input_rows_kernel<11><<<grid_for(rows), 256, 0, st>>>(dz, w, din, M, Cin, Cout);
    else if (H == 5 && Cout % 8 == 0 && Cin % 32 == 0)
        conv5x5_gemm_kernel<true, 4><<<dim3((M + 3) / 4, Cin / 32), 160, 0, st>>>(dz, w, nullptr, din, M, Cout, Cin, Cin);
    else if (H == 5) conv3x3_bwd_input_rows_kernel<5><<<grid_for(rows), 256, 0, st>>>(dz, w, din, M, Cin, Cout);
    else if (H == 2 && Cout % 8 == 0 && Cin % 32 == 0 && ((reinterpret_cast<uintptr_t>(dz) | reinterpret_cast<uintptr_t>(din)) & 15u) == 0)
        conv2x2_gemm_kernel<true><<<dim3((M + 15) / 16, Cin / 32), 256, 0, st>>>(dz, w, nullptr, din, M, Cout, Cin, Cin);
    else if (H == 2 && ((reinterpret_cast<uintptr_t>(dz) | reinterpret_cast<uintptr_t>(din)) & 15u) == 0)
        conv3x3_bwd_input_2x2_kernel<<<grid_for((long long)((M + 3) / 4) * Cin), 256, 0, st>>>(dz, w, din, M, Cin, Cout);
    else if (H == 2) conv3x3_bwd_input_rows_kernel<2><<<grid_for(rows), 256, 0, st>>>(dz, w, din, M, Cin, Cout);
    else conv3x3_bwd_input_kernel<<<grid_for(rows * H), 256, 0, st>>>(dz, w, din, M, Cin, Cout, H);
}
static void launch_conv_bwd_weight(const float* dz, const float* in, float* partial, float* partial_b, int M, int Cin,
                                   int Cout, int H, int imgs_per_chunk, int chunks, cudaStream_t st) {
    const int nP = Cout * Cin;
    const dim3 grid((nP + Cout + 127) / 128, chunks);
    if (H == 11) conv3x3_bwd_weight_taps_kernel<11><<<grid, 128, 0, st>>>(dz, in, partial, partial_b, M, Cin, Cout, imgs_per_chunk);
    else if (H == 5) conv3x3_bwd_weight_taps_kernel<5><<<grid, 128, 0, st>>>(dz, in, partial, partial_b, M, Cin, Cout, imgs_per_chunk);
    else if (H == 2) conv3x3_bwd_weight_taps_kernel<2><<<grid, 128, 0, st>>>(dz, in, partial, partial_b, M, Cin, Cout, imgs_per_chunk);
    else
        conv3x3_bwd_weight_kernel<<<dim3((nP * 9 + Cout + 255) / 256, chunks), 256, 0, st>>>(dz, in, partial, partial_b, M, Cin,
                                                                                         Cout, H, imgs_per_chunk);
}

}  // namespace gpp

using namespace gpp;

extern "C" size_t gpp_planner_train_workspace_bytes(int B, int N, int K) {
    if (B <= 0 || N <= 0 || K <= 0) return 0;
    return train_layout(B, N, K).total * sizeof(float);
}

extern "C" int gpp_planner_train_forward(const gpp_planner_weights* w, const gpp_planner_bn_state* bn, float momentum,
                                         const float* x, const void* S, int s_is_f64, float* logits, void* workspace,
                                         int B, int N, int K, void* stream) {
    GPP_REQUIRE(w && x && S && logits && workspace, GPP_ERR_INVALID, "planner_train_forward: null pointer");
    GPP_REQUIRE(B >= 1 && N >= 1 && N <= 64 && K >= 1, GPP_ERR_INVALID, "planner_train_forward: bad sizes B=%d N=%d K=%d", B, N, K);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const TrainWs L = train_layout(B, N, K);
    float* ws = reinterpret_cast<float*>(workspace);
    const int M = B * N;
    const float* in = x;
    for (int l = 0; l < 5; ++l) {
        const int Cin = kC[l], Cout = kC[l + 1], H = kH[l], HW = H * H;
        const long long total = (long long)M * Cout * HW;
        float* z = ws + L.z[l];
        float* a = ws + L.a[l];
        launch_conv_fwd(in, w->conv_w[l], w->conv_b[l], z, M, Cin, Cout, H, st);
        GPP_LAUNCH_CHECK();
        const bool pool = pooled_after(l);
        bn_stats_kernel<<<N * Cout, 128, 0, st>>>(z, ws + L.mean[l], ws + L.var[l], ws + L.invstd[l], B, N, Cout, HW, 1e-5f,
                                                  w->bn_w[l], w->bn_b[l], a, pool ? ws + L.p[l] : nullptr, H,
                                                  pool ? pooled_hw(l) : 0);
        GPP_LAUNCH_CHECK();
        (void)total;
        if (bn && bn->running_mean[l] && bn->running_var[l]) {
            bn_running_kernel<<<(Cout + 127) / 128, 128, 0, st>>>(ws + L.mean[l], ws + L.var[l], bn->running_mean[l],
                                                                  bn->running_var[l], N, Cout, B * HW, momentum);
            GPP_LAUNCH_CHECK();
        }
        in = pool ? ws + L.p[l] : a;
    }
    linear128_fwd_rowwarp_kernel<<<(M + 7) / 8, 256, 0, st>>>(in, w->compress_w, w->compress_b, ws + L.feat, M, 1);
    GPP_LAUNCH_CHECK();
    int rc = gpp_graph_filter_forward(ws + L.feat, S, s_is_f64, w->gf_w, w->gf_b, ws + L.shared, B, N, 128, 128, K,
                                      GPP_NODE_MAJOR, GPP_NODE_MAJOR, 1, ws + L.gf_fwd, stream);
    if (rc) return rc;
    action_fwd_kernel<<<(M * 5 + 255) / 256, 256, 0, st>>>(ws + L.shared, w->action_w, w->action_b, logits, B, N);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

extern "C" int gpp_planner_train_backward(const gpp_planner_weights* w, const float* x, const void* S, int s_is_f64,
                                          const float* dlogits, void* workspace, const gpp_planner_grads* g, int B,
                                          int N, int K, void* stream) {
    GPP_REQUIRE(w && x && S && dlogits && workspace && g, GPP_ERR_INVALID, "planner_train_backward: null pointer");
    GPP_REQUIRE(B >= 1 && N >= 1 && N <= 64 && K >= 1, GPP_ERR_INVALID, "planner_train_backward: bad sizes");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const TrainWs L = train_layout(B, N, K);
    float* ws = reinterpret_cast<float*>(workspace);
    const int M = B * N;
    // ---- action MLP
    action_bwd_input_kernel<<<grid_for((long long)M * 128), 256, 0, st>>>(dlogits, w->action_w, ws + L.dshared, B, N);
    GPP_LAUNCH_CHECK();
    {
        double* apart = reinterpret_cast<double*>(ws + L.partial);      // free until the weight-gradient kernels below
        action_bwd_weight_partial_kernel<<<kActChunks, 128, 0, st>>>(dlogits, ws + L.shared, apart, B, N);
        GPP_LAUNCH_CHECK();
        action_bwd_weight_reduce_kernel<<<6, 128, 0, st>>>(apart, g->action_w, g->action_b);
        GPP_LAUNCH_CHECK();
    }
    // ---- graph filter (+ReLU): fused kernels
    int rc = gpp_graph_filter_backward(ws + L.dshared, ws + L.shared, ws + L.feat, S, s_is_f64, w->gf_w, ws + L.dfeat,
                                       g->gf_w, g->gf_b, B, N, 128, 128, K, GPP_NODE_MAJOR, GPP_NODE_MAJOR, 1,
                                       ws + L.gf_bwd, stream);
    if (rc) return rc;
    // ---- compress MLP (+ReLU)
    const float* lin_in = ws + L.p[4];
    relu_mask_kernel<<<grid_for((long long)M * 128), 256, 0, st>>>(ws + L.dfeat, ws + L.feat, (long long)M * 128);
    GPP_LAUNCH_CHECK();
    {
        const int rpc = (M + L.chunks - 1) / L.chunks;
        const int used = (M + rpc - 1) / rpc;
        linear_bwd_weight_kernel<<<dim3((128 * 128 + 128 + 255) / 256, used), 256, 0, st>>>(
            ws + L.dfeat, lin_in, ws + L.partial, ws + L.partial_b, M, 128, 128, rpc);
        GPP_LAUNCH_CHECK();
        reduce_chunks_kernel<<<(128 * 128 + 255) / 256, 256, 0, st>>>(ws + L.partial, g->compress_w, used, 128 * 128);
        GPP_LAUNCH_CHECK();
        reduce_chunks_kernel<<<1, 128, 0, st>>>(ws + L.partial_b, g->compress_b, used, 128);
        GPP_LAUNCH_CHECK();
    }
    float* dcur = ws + L.dbuf0;      // gradient w.r.t. the current layer's output (post-pool if pooled)
    float* dnext = ws + L.dbuf1;
    linear_bwd_input_kernel<<<grid_for((long long)M * 128), 256, 0, st>>>(ws + L.dfeat, w->compress_w, dcur, M, 128, 128);
    GPP_LAUNCH_CHECK();
    // ---- conv stack, last layer first
    for (int l = 4; l >= 0; --l) {
        const int Cin = kC[l], Cout = kC[l + 1], H = kH[l], HW = H * H;
        const long long total = (long long)M * Cout * HW;
        const float* z = ws + L.z[l];
        const float* a = ws + L.a[l];
        float* da = dcur;
        if (pooled_after(l)) {
            const int Hp = pooled_hw(l);
            maxpool2_bwd_kernel<<<grid_for(total), 256, 0, st>>>(a, dcur, dnext, total, H, Hp);
            GPP_LAUNCH_CHECK();
            da = dnext;
            float* t = dcur; dcur = dnext; dnext = t;
        }
        double* s1 = reinterpret_cast<double*>(ws + L.s1);
        double* s2 = reinterpret_cast<double*>(ws + L.s2);
        bn_bwd_reduce_kernel<<<N * Cout, 128, 0, st>>>(da, a, z, ws + L.mean[l], ws + L.invstd[l], w->bn_w[l], s1, s2, B, N,
                                                       Cout, HW);
        GPP_LAUNCH_CHECK();
        bn_param_grad_kernel<<<(Cout + 127) / 128, 128, 0, st>>>(s1, s2, g->bn_w[l], g->bn_b[l], N, Cout);
        GPP_LAUNCH_CHECK();
        // da now holds dz
        const float* lin = (l == 0) ? x : (pooled_after(l - 1) ? ws + L.p[l - 1] : ws + L.a[l - 1]);
        {
            const int ipc = (M + L.chunks - 1) / L.chunks;
            const int used = (M + ipc - 1) / ipc;
            const int nW = Cout * Cin * 9;
            launch_conv_bwd_weight(da, lin, ws + L.partial, ws + L.partial_b, M, Cin, Cout, H, ipc, used, st);
            GPP_LAUNCH_CHECK();
            reduce_chunks_kernel<<<(nW + 255) / 256, 256, 0, st>>>(ws + L.partial, g->conv_w[l], used, nW);
            GPP_LAUNCH_CHECK();
            reduce_chunks_kernel<<<1, 128, 0, st>>>(ws + L.partial_b, g->conv_b[l], used, Cout);
            GPP_LAUNCH_CHECK();
        }
        if (l > 0) {
            launch_conv_bwd_input(da, w->conv_w[l], dnext, M, Cin, Cout, H, st);
            GPP_LAUNCH_CHECK();
            float* t = dcur; dcur = dnext; dnext = t;
        }
    }
    return GPP_OK;
}

// ---------------------------------------------------------------------------------------
// Fused training loss (SURVEY.md section 8 row f3): replaces the per-agent loop of
// agents/decentralplannerlocal.py:305-312 -- loss = (1/N) sum_i CrossEntropy(predict[i], argmax(target[:, i])) -- and
// the backward seed d loss / d logits, in ONE launch on the contiguous [N,B,5] logits (the reference's loop is N
// log-softmax + NLL + mean kernels forward and as many backward).  One block, fp64 partial sums combined in a fixed
// order: deterministic.  argmax = first maximum, as torch.max(., 1)[1] on a one-hot row.
// ---------------------------------------------------------------------------------------
namespace gpp {
template <typename T>
__global__ void __launch_bounds__(1024) ce_loss_kernel(const float* __restrict__ logits, const T* __restrict__ target,
                                                       float* __restrict__ loss, float* __restrict__ dlogits, int B, int N,
                                                       float grad_scale) {
    __shared__ double red[32];
    const int rows = N * B;
    const float inv = 1.f / (float)rows;
    double acc = 0.0;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) {
        const int n = r / B, b = r - n * B;
        const float* lp = logits + (size_t)r * 5;
        const T* tp = target + ((size_t)b * N + n) * 5;            // target is [B,N,5]
        int cls = 0;
        T best = tp[0];
#pragma unroll
        for (int q = 1; q < 5; ++q)
            if (tp[q] > best) { best = tp[q]; cls = q; }
        float v[5], mx = lp[0];
#pragma unroll
        for (int q = 0; q < 5; ++q) { v[q] = lp[q]; mx = fmaxf(mx, v[q]); }
        float sum = 0.f, e[5];
#pragma unroll
        for (int q = 0; q < 5; ++q) { e[q] = expf(v[q] - mx); sum += e[q]; }
        const float lse = mx + logf(sum);
        acc += (double)(lse - v[cls]);
        if (dlogits) {
            const float rs = 1.f / sum;
#pragma unroll
            for (int q = 0; q < 5; ++q) dlogits[(size_t)r * 5 + q] = (e[q] * rs - (q == cls ? 1.f : 0.f)) * inv * grad_scale;
        }
    }
    // fixed-order reduction: lanes by xor-butterfly (same tree every run), warps in index order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) t += red[wv];
        *loss = (float)(t / (double)rows);
    }
}
}  // namespace gpp

extern "C" int gpp_planner_ce_loss(const float* logits, const void* target_onehot, int target_is_i64, float* loss,
                                   float* dlogits, float grad_scale, int B, int N, void* stream) {
    GPP_REQUIRE(logits && target_onehot && loss, GPP_ERR_INVALID, "planner_ce_loss: null pointer");
    GPP_REQUIRE(B >= 1 && N >= 1, GPP_ERR_INVALID, "planner_ce_loss: bad sizes B=%d N=%d", B, N);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (target_is_i64)
        ce_loss_kernel<long long><<<1, 1024, 0, st>>>(logits, reinterpret_cast<const long long*>(target_onehot), loss, dlogits,
                                                      B, N, grad_scale);
    else
        ce_loss_kernel<float><<<1, 1024, 0, st>>>(logits, reinterpret_cast<const float*>(target_onehot), loss, dlogits, B, N,
                                                  grad_scale);
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}

// debug: single training kernels for unit tests (tests/ only)
//   op 0: conv3x3_fwd (a = in, b = w, c = bias)      op 1: conv3x3_bwd_input (a = dz, b = w)
//   op 2: maxpool2_bwd (a = act, b = dp)           op 3: conv3x3 weight/bias gradient (a = dz, b = in) -> dW | db
extern "C" int gpp_debug_train_kernel(int op, const float* a, const float* b, const float* c, float* out, int M,
                                      int Cin, int Cout, int H, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (op == 0) {
        launch_conv_fwd(a, b, c, out, M, Cin, Cout, H, st);
    } else if (op == 1) {
        launch_conv_bwd_input(a, b, out, M, Cin, Cout, H, st);
    } else if (op == 2) {
        const long long total = (long long)M * Cout * H * H;
        maxpool2_bwd_kernel<<<grid_for(total), 256, 0, st>>>(a, b, out, total, H, H / 2);
    } else if (op == 3) {
        // conv weight + bias gradient exactly as the training step computes it: per-chunk partial sums, then the
        // fixed-order chunk reduction.  out = dW [Cout][Cin][3][3] followed by db [Cout].
        const int chunks = M < 64 ? M : 64;
        const int ipc = (M + chunks - 1) / chunks;
        const int used = (M + ipc - 1) / ipc;
        const int nW = Cout * Cin * 9;
        float* scratch = nullptr;
        GPP_CUDA_OK(cudaMallocAsync(&scratch, sizeof(float) * ((size_t)used * nW + (size_t)used * Cout), st));
        float* partial_b = scratch + (size_t)used * nW;
        launch_conv_bwd_weight(a, b, scratch, partial_b, M, Cin, Cout, H, ipc, used, st);
        GPP_LAUNCH_CHECK();
        reduce_chunks_kernel<<<(nW + 255) / 256, 256, 0, st>>>(scratch, out, used, nW);
        GPP_LAUNCH_CHECK();
        reduce_chunks_kernel<<<(Cout + 127) / 128, 128, 0, st>>>(partial_b, out + nW, used, Cout);
        GPP_CUDA_OK(cudaFreeAsync(scratch, st));
    } else {
        set_error("debug_train_kernel: unknown op %d", op);
        return GPP_ERR_INVALID;
    }
    GPP_LAUNCH_CHECK();
    return GPP_OK;
}
