/*
 * gnnpp_b200_debug.h -- test / profiling hooks of libgnnpp_b200.so.  NOT part of the drop-in boundary
 * (include/gnnpp_b200.h): nothing here replaces a reference interface; tests/ and profiles/ use these to
 * exercise single kernels and to read in-kernel phase timers.  All switches default to off.
 */
#ifndef GNNPP_B200_DEBUG_H
#define GNNPP_B200_DEBUG_H

#ifdef __cplusplus
extern "C" {
#endif

/* Process-wide debug switches (replace the round-1 environment variables):
 *   "gf_timing" / "tc_timing" / "fe_timing"  != 0: the CUDA-core filter / tensor-core kernels / CUDA-core feature
 *                 kernel accumulate per-phase clock64() totals, read with the gpp_debug_*_timing calls below
 *   "no_pdl"     != 0: planner kernels are launched without programmatic dependent launch
 *   "gf_mode"    kernel choice of the standalone gpp_graph_filter_forward: 0 auto, 1 CUDA-core, 2 wgmma 3xTF32,
 *                3 wgmma pair fp16-split
 *   "pair_ablate" (performance experiments only, results are wrong) bit mask for the CTA-pair kernel: 1 skip the
 *                propagations, 2 skip the operand stores, 4 skip the x loads, 8 skip the y stores
 *   "stage_mode" (probe) input staging of gpp_planner_forward_host_async: 0 copy engine (production), != 0 the copy
 *                kernel that pulls pinned memory with 16-byte loads
 *   "lanes"      (probe) compute lanes used by the pipelined entry points: 1 .. 4, 0 = all four */
int gpp_debug_set_option(const char* name, int value);

/* Test hook for the wgmma plumbing: D[128][128] = A[128][32] . B[128][32]^T on the tensor cores
 * (A, B tf32-representable fp32, row-major, device memory). */
int gpp_debug_umma_selftest(const float* A, const float* B, float* D, void* stream);

/* Debug: per-phase cycle totals of the 3xTF32 tensor-core filter kernel (filled only when the "tc_timing" option is set): staging loop, wait for U_k, (unused), propagation, stores, tiles. */
int gpp_debug_tc_timing(unsigned long long* out6);
/* Per-role cycle totals of the fp16-split pair filter kernel ("tc_timing"): [0..3] producer warp 0 of every CTA: wait
 * for S, wait for a ring slot, item work, items; [4..6] leader MMA threads: wait for operands, wait for the accumulator,
 * loop total; [7..8] epilogue warp 0: wait, work; [9..10] scout: wait, work; [11] tile pairs; [12] kernel cycles
 * (thread 0 of every CTA); [13] leader start-up until the taps landed; [14] CTAs. */
int gpp_debug_pair_timing(unsigned long long* out16);
/* Same for block 0 of the CUDA-core filter kernel ("gf_timing"): prologue, x/S staging,
 * propagation, tap contraction, epilogue, action MLP + column-half merge. */
int gpp_debug_gf_timing(unsigned long long* out6);
/* Same for the 3xTF32 tensor-core feature extractor: [3*L + {0,1,2}] = layer L staging loop / wait for MMAs / epilogue,
 * [18] = agent tiles (thread 0 of every CTA). */
int gpp_debug_feature_tc_timing(unsigned long long* out20);
/* feature_mma_kernel phase timers of thread 0 of block 0 ("tc_timing" option on): [6..11] waiting for filter chunks
 * per layer, [12..17] MMAs per layer, [18] tiles, [19] input conversion, [26..31] epilogue work per layer; 40 entries
 * (the others stay 0); cycles, cleared by the call */
int gpp_debug_feature_mma_timing(unsigned long long* out40);
/* Block 0 of the CUDA-core feature extractor ("fe_timing"): input staging, conv0, conv1,
 * conv2, conv3, conv4, compress MLP + store. */
int gpp_debug_feature_timing(unsigned long long* out7);
/* Single kernels of the native training path (tests/test_gpu_train_ops.py): op 0 conv3x3 forward (a = input, b = filters,
 * c = bias), op 1 conv3x3 input gradient (a = dz, b = filters), op 2 max-pool gradient (a = activation, b = pooled grad), op 3 conv3x3
 * weight + bias gradient (a = dz, b = input; out = dW [Cout,Cin,3,3] followed by db [Cout]). */
int gpp_debug_train_kernel(int op, const float* a, const float* b, const float* c, float* out, int M, int Cin, int Cout,
                           int H, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GNNPP_B200_DEBUG_H */
