/* CPU ORACLE (plain C) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Restates the reference's per-sample-GSO graph filter, BatchLSIGF
 * (gnn_pathplanning/utils/graphUtils/graphML.py:2273-2367), element by element:
 *     z_0 = x ;  z_k[g,n] = sum_m z_{k-1}[g,m] * (float)S[m,n]        (:2350, right-multiply)
 *     y[f,n] = sum_{k,g} h[f,0,k,g] * z_k[g,n] + b[f]                  (:2361-2366)
 * Two variants: f32 storage of every z_k like the reference's float32 tensors with f64
 * accumulation inside each dot product ("gf_oracle_f32"), and all-f64 ("gf_oracle_f64") used
 * to bound rounding error of both the reference and the CUDA kernels.
 * Pinned against the reference-generated golden vectors by tests/test_oracle_golden.py.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this. */
#include <stdlib.h>
#include <string.h>

/* x [B,G,N] f32, S [B,N,N] f32 or f64 (s_is_f64), h [F,K,G] f32 (E = 1), b [F] or NULL,
 * y [B,F,N] (f32 for _f32, f64 for _f64).  Returns 0, or -1 on allocation failure. */
static int run(const float* x, const void* S, int s_is_f64, const float* h, const float* b,
               void* y, int y_is_f64, int B, int N, int G, int F, int K, int z_f32) {
    double* z = (double*)malloc(sizeof(double) * (size_t)K * G * N);
    double* Sm = (double*)malloc(sizeof(double) * (size_t)N * N);
    if (!z || !Sm) { free(z); free(Sm); return -1; }
    for (int bi = 0; bi < B; ++bi) {
        for (int i = 0; i < N * N; ++i) {
            /* the reference casts the GSO to float32 before every product (S.float(), :2350) */
            float sf = s_is_f64 ? (float)((const double*)S)[(size_t)bi * N * N + i]
                                : ((const float*)S)[(size_t)bi * N * N + i];
            Sm[i] = (double)sf;
        }
        for (int i = 0; i < G * N; ++i) z[i] = (double)x[(size_t)bi * G * N + i];
        for (int k = 1; k < K; ++k)
            for (int g = 0; g < G; ++g)
                for (int n = 0; n < N; ++n) {
                    double acc = 0.0;
                    for (int m = 0; m < N; ++m) acc += z[((size_t)(k - 1) * G + g) * N + m] * Sm[m * N + n];
                    z[((size_t)k * G + g) * N + n] = z_f32 ? (double)(float)acc : acc;
                }
        for (int f = 0; f < F; ++f)
            for (int n = 0; n < N; ++n) {
                double acc = 0.0;
                for (int j = 0; j < K * G; ++j) acc += (double)h[(size_t)f * K * G + j] * z[(size_t)j * N + n];
                if (b) acc += (double)b[f];
                size_t o = ((size_t)bi * F + f) * N + n;
                if (y_is_f64) ((double*)y)[o] = acc; else ((float*)y)[o] = (float)acc;
            }
    }
    free(z); free(Sm);
    return 0;
}

int gf_oracle_f32(const float* x, const void* S, int s_is_f64, const float* h, const float* b,
                  float* y, int B, int N, int G, int F, int K) {
    return run(x, S, s_is_f64, h, b, y, 0, B, N, G, F, K, 1);
}

int gf_oracle_f64(const float* x, const void* S, int s_is_f64, const float* h, const float* b,
                  double* y, int B, int N, int G, int F, int K) {
    return run(x, S, s_is_f64, h, b, y, 1, B, N, G, F, K, 0);
}
