// Whole-planner inference for sm_90a: host side of the C ABI (include/gnnpp_b200.h).
//
// Replaces DecentralPlannerNet.addGSO + forward in eval mode
// (gnn_pathplanning/graphs/models/decentralplanner.py:266-318) with two kernels:
//   feature_kernel  (feature.cu)       per-agent CNN + compress MLP, agents tiled onto CTAs
//   gf_fwd_kernel   (graph_filter.cu)  K-tap graph filter + ReLU + action MLP, logits out
// plus the one-off parameter re-layout (k-major filters, eval BatchNorm folded to scale/shift).
#include "common.cuh"
#include "feature.cuh"

#include <utility>
#include "../../include/gnnpp_b200_debug.h"

#include <stdarg.h>
#include <string.h>

#include <vector>

namespace gpp {

// ---- error / bookkeeping ----------------------------------------------------------------
static thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};     // process-wide: autograd runs the backward on its own thread

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached[kMaxDevices] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev >= 0 && dev < kMaxDevices && cached[dev] > 0) return cached[dev];
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    if (dev >= 0 && dev < kMaxDevices) cached[dev] = n;
    return n;
}

static int g_debug_options[DBG_COUNT] = {};
int debug_option(int which) { return (which >= 0 && which < DBG_COUNT) ? g_debug_options[which] : 0; }

// internal launchers from graph_filter.cu
int launch_transpose_taps(const float* w, float* wt, int F, int KG, cudaStream_t st);
int launch_split_taps(const float* wt, float* ws, int KG, cudaStream_t st);
int launch_gf_forward_fast(const float* x, const void* S, int s_is_f64, const float* wt,
                           const float* bias, float* y, const float* wa, const float* ba,
                           float* logits, int B, int N, int K, int x_layout, int y_layout,
                           int relu, int allow_bulk, float* lpart, unsigned int* tickets, const float* wsplit,
                           int pdl, cudaStream_t st);
// tensor-core path (graph_filter_tc.cu)
size_t gf_tc_image_floats(int K);
int gf_tc_tile_samples(int N, int K);
int launch_prep_umma_taps(const float* w, float* img, int K, cudaStream_t st);
int launch_gf_forward_tc(const float* x, const void* S, int s_is_f64, const float* wimg, const float* bias,
                         float* y, const float* wa, const float* ba, float* logits, int B, int N, int K,
                         int relu, int allow_bulk, cudaStream_t st);

// fp16-split wgmma pair path (graph_filter_pair.cu)
size_t gf_pair_image_bytes(int K);
bool gf_pair_supported(int N, int K);
int launch_prep_pair_taps(const float* w, void* img, int K, cudaStream_t st);
int launch_gf_forward_pair(const float* x, const void* S, int s_is_f64, const void* wimg, const float* bias, float* y,
                           const float* wa_host, const float* ba_host, float* logits, int B, int N, int K, int relu,
                           cudaStream_t st);

// Host -> device staging as a kernel (probe path of gpp_planner_forward_host_async, "stage_mode" debug option; the
// production path uses the copy engine): a few CTAs pull pinned (device-mapped) host memory over PCIe with 16-byte loads
// and store it to HBM; n16 = number of 16-byte units, tail bytes separately.
// both inputs of a step in one launch: blocks [0, gridDim.x - 1) copy x, the last block copies S
struct StagePair {
    const uint4* src[2];
    uint4* dst[2];
    size_t n16[2];
    int tail[2];
};
__global__ void __launch_bounds__(256) stage_h2d_pair_kernel(const StagePair sp) {
    const int which = blockIdx.x == gridDim.x - 1 ? 1 : 0;
    const int nb = which ? 1 : gridDim.x - 1, b = which ? 0 : blockIdx.x;
    const uint4* __restrict__ src = sp.src[which];
    uint4* __restrict__ dst = sp.dst[which];
    const size_t n16 = sp.n16[which], stride = (size_t)nb * blockDim.x;
    for (size_t i = (size_t)b * blockDim.x + threadIdx.x; i < n16; i += stride) dst[i] = src[i];
    if (b == 0 && (int)threadIdx.x < sp.tail[which])
        reinterpret_cast<unsigned char*>(dst + n16)[threadIdx.x] = reinterpret_cast<const unsigned char*>(src + n16)[threadIdx.x];
}

// tensor-core feature extractor (feature_tc.cu)
size_t feature_tc_image_floats(int L);
int launch_prep_feature_tc(const float* w, float* img, int L, cudaStream_t st);
int launch_feature_tc_kernel(const FeArgs& fa, const float* const* imgs, cudaStream_t st);
int debug_feature_tc_timing(unsigned long long* out20);
// small-batch wgmma graph filter + action MLP (graph_filter_small.cu)
size_t gf_small_arena_bytes(int K);
bool gf_small_supported(int N, int K);
int launch_prep_gf_small(const float* w, float* arena, int K, cudaStream_t st);
int launch_gf_forward_small(const float* x, const void* S, int s_is_f64, const float* arena, const float* bias,
                            const float* wa, const float* ba, float* logits, int B, int K, int pdl, cudaStream_t st);
// im2col-free fp16-split tensor-core feature extractor (feature_mma.cu)
size_t feature_mma_arena_floats();
int launch_prep_feature_mma(const float* const* conv_w, const float* compress_w, const float* const* sc,
                            const float* const* sh, const float* b5, float* arena, cudaStream_t st);
int launch_feature_mma_kernel(const FeArgs& fa, const float* arena, int x_bulk, cudaStream_t st);
int debug_feature_mma_timing(unsigned long long* out32);
int debug_feature_timing(unsigned long long* out7);

// scale = gamma / sqrt(var + eps);  shift = (conv_bias - mean) * scale + beta
__global__ void fold_bn_kernel(const float* conv_b, const float* g, const float* b, const float* mean,
                               const float* var, float* sc, float* sh, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C) return;
    const float s = g[i] / sqrtf(var[i] + 1e-5f);
    sc[i] = s;
    sh[i] = (conv_b[i] - mean[i]) * s + b[i];
}

}  // namespace gpp

using namespace gpp;

static const int kConvC[6] = {3, 32, 32, 64, 64, 128};
static const int IN_PIX = 3 * 11 * 11;

constexpr int kLanes = 4;        // compute lanes of the pipelined host-buffer path
constexpr int kStageSlots = 8;   // device staging slots of the pipelined host-buffer path (steps in flight)

struct gpp_planner {
    int K;
    int device;          // CUDA device ordinal the handle (arena, scratch, streams) lives on
    cudaStream_t last_stream;    // stream of the most recent forward / weight staging: a call on another stream first
    bool last_stream_valid;      // waits for it (the feature workspace and the filter's scratch are shared per handle)
    cudaEvent_t order_event;
    float* arena;        // prepared weights
    size_t off_w[6];     // conv0..4 k-major, compress k-major
    size_t off_sc[5], off_sh[5];
    size_t off_b5, off_gfw, off_gfws, off_gfb, off_wa, off_ba, off_gfimg, off_gfpair, arena_floats;
    float wa_host[5 * 128 + 8];   // host copy of the action MLP: the CTA-pair filter kernel takes it as kernel parameters
    bool pdl_ok;         // the kernels before the next forward in its stream only wrote what it reads after its
                         // griddepcontrol.wait (false right after the weights were re-staged)
    int gf_mode;         // 0 auto, 1 CUDA-core kernel, 2 wgmma 3xTF32 kernel, 3 wgmma pair fp16-split kernel
    int fe_mode;         // feature extractor: 0 auto, 1 CUDA-core kernel, 2 wgmma 3xTF32 kernel, 3 wgmma fp16-split kernel
    size_t off_fmma;     // images + constants of the fp16-split kernel
    size_t off_gfsmall;  // tap images of the small-batch wgmma graph filter
    size_t off_fimg[6];  // wgmma filter chunk images of conv0..4 and the compress MLP
    bool weights_set;
    float* raw;          // device staging for host-provided parameters
    size_t raw_floats;
    // extra compute lanes of the pipelined host path (gpp_planner_forward_host_async rotates over kLanes streams so that
    // the feature kernel of one batch overlaps the graph-filter kernel of the batch before it and the idle SMs of a
    // 640-agent launch take the next batch's tiles): own stream and scratch each; swapped in for the duration of a call by
    // LaneGuard.  Lane 0 is the handle's own stream and scratch.
    cudaStream_t lane_stream[kLanes - 1];
    bool lanes_active;   // inside gpp_planner_forward_host_async
    float* lane_feat[kLanes - 1]; size_t lane_feat_rows[kLanes - 1]; float* lane_lpart[kLanes - 1];
    size_t lane_lpart_rows[kLanes - 1]; bool lane_pdl_ok[kLanes - 1];
    float* feat;         // [rows][128] workspace
    size_t feat_rows;
    const void* alias_host[16];   // pinned host buffers seen by the async entry point and their device aliases
    void* alias_dev[16];
    unsigned alias_next;
    float* gf_lpart;     // [2][rows][5] partial logits + [rows] tile tickets of the column-split filter launch
    size_t gf_lpart_rows;
    // host-buffer path
    cudaStream_t stream;
    float* d_x;
    size_t d_x_floats;
    void* d_S;
    size_t d_S_bytes;
    float* d_logits;
    size_t d_logits_floats;
    // asynchronous host-buffer calls: completion tickets + double-buffered H2D staging on a copy stream
    cudaEvent_t tickets[16];
    cudaEvent_t ready[16];       // gpp_planner_forward_async: the caller's stream at submission
    unsigned long long next_ticket;
    cudaStream_t copy_stream;
    float* a_x[kStageSlots];
    size_t a_x_floats[kStageSlots];
    void* a_S[kStageSlots];
    size_t a_S_bytes[kStageSlots];
    cudaEvent_t copied[kStageSlots];
    // per-kernel event log (roofline report)
    bool profiling;
    std::vector<cudaEvent_t>* events;   // triples: start, after feature kernel, after filter kernel
    size_t events_used;
};

extern "C" const char* gpp_last_error(void) { return gpp::g_err; }
extern "C" int gpp_abi_version(void) { return 1; }
extern "C" unsigned long long gpp_launch_count(void) { return gpp::g_launches.load(); }
extern "C" void gpp_reset_launch_count(void) { gpp::g_launches.store(0); }

extern "C" int gpp_device_info(int* sms, int* cc_major, int* cc_minor) {
    int dev = 0;
    GPP_CUDA_OK(cudaGetDevice(&dev));
    cudaDeviceProp p;
    GPP_CUDA_OK(cudaGetDeviceProperties(&p, dev));
    if (sms) *sms = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    return GPP_OK;
}

extern "C" int gpp_planner_create(gpp_planner** out, int K) {
    GPP_REQUIRE(out, GPP_ERR_INVALID, "planner_create: null out pointer");
    GPP_REQUIRE(K >= 1 && K <= 8, GPP_ERR_UNSUPPORTED, "planner_create: K=%d outside [1,8]", K);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("planner_create: no CUDA device visible");
        return GPP_ERR_NODEVICE;
    }
    gpp_planner* p = new gpp_planner();
    memset(p, 0, sizeof(*p));
    p->K = K;
    if (cudaGetDevice(&p->device) != cudaSuccess) p->device = 0;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off += (n + 63) / 64 * 64; return o; };
    for (int l = 0; l < 5; ++l) p->off_w[l] = take((size_t)kConvC[l] * 9 * kConvC[l + 1]);
    p->off_w[5] = take(128 * 128);
    for (int l = 0; l < 5; ++l) { p->off_sc[l] = take(kConvC[l + 1]); p->off_sh[l] = take(kConvC[l + 1]); }
    p->off_b5 = take(128);
    p->off_gfw = take((size_t)K * 128 * 128);
    p->off_gfws = take((size_t)K * 128 * 128);       // the same taps, column halves contiguous
    p->off_gfb = take(128);
    p->off_wa = take(5 * 128);
    p->off_ba = take(64);
    p->off_gfimg = take(gf_tc_image_floats(K));      // pre-split, pre-swizzled wgmma B-operand chunks
    p->off_gfpair = take(K <= 3 ? gf_pair_image_bytes(K) / 4 + 16 : 16);
    for (int l = 0; l < 6; ++l) p->off_fimg[l] = take(feature_tc_image_floats(l));
    p->off_fmma = take(feature_mma_arena_floats());
    p->off_gfsmall = take(K <= 3 ? gf_small_arena_bytes(K) / 4 + 16 : 16);
    p->arena_floats = off;
    if (cudaMalloc(&p->arena, sizeof(float) * off) != cudaSuccess) {
        set_error("planner_create: cudaMalloc(%zu) failed", sizeof(float) * off);
        delete p;
        return GPP_ERR_CUDA;
    }
    if (cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) != cudaSuccess) {
        set_error("planner_create: stream creation failed");
        cudaFree(p->arena);
        delete p;
        return GPP_ERR_CUDA;
    }
    *out = p;
    return GPP_OK;
}

extern "C" void gpp_planner_destroy(gpp_planner* p) {
    if (!p) return;
    cudaFree(p->arena);
    cudaFree(p->raw);
    cudaFree(p->feat);
    cudaFree(p->gf_lpart);
    for (int l = 0; l < kLanes - 1; ++l) {
        cudaFree(p->lane_feat[l]);
        cudaFree(p->lane_lpart[l]);
        if (p->lane_stream[l]) cudaStreamDestroy(p->lane_stream[l]);
    }
    cudaFree(p->d_x);
    cudaFree(p->d_S);
    cudaFree(p->d_logits);
    if (p->stream) cudaStreamDestroy(p->stream);
    if (p->order_event) cudaEventDestroy(p->order_event);
    for (int i = 0; i < 16; ++i) {
        if (p->tickets[i]) cudaEventDestroy(p->tickets[i]);
        if (p->ready[i]) cudaEventDestroy(p->ready[i]);
    }
    for (int i = 0; i < kStageSlots; ++i) {
        cudaFree(p->a_x[i]);
        cudaFree(p->a_S[i]);
        if (p->copied[i]) cudaEventDestroy(p->copied[i]);
    }
    if (p->copy_stream) cudaStreamDestroy(p->copy_stream);
    if (p->events) {
        for (cudaEvent_t e : *p->events) cudaEventDestroy(e);
        delete p->events;
    }
    delete p;
}

extern "C" int gpp_planner_set_graph_filter_mode(gpp_planner* p, int mode) {
    GPP_REQUIRE(p && mode >= 0 && mode <= 3, GPP_ERR_INVALID, "planner_set_graph_filter_mode: mode must be 0, 1, 2 or 3");
    p->gf_mode = mode;
    return GPP_OK;
}

// debug: per-layer {staging loop, wait for MMAs, epilogue} cycle totals of feature_tc_kernel + tiles at [18]
extern "C" int gpp_debug_feature_tc_timing(unsigned long long* out20) { return debug_feature_tc_timing(out20); }
extern "C" int gpp_debug_feature_timing(unsigned long long* out7) { return debug_feature_timing(out7); }
extern "C" int gpp_debug_feature_mma_timing(unsigned long long* out32) { return debug_feature_mma_timing(out32); }

// debug switches (include/gnnpp_b200_debug.h)
extern "C" int gpp_debug_set_option(const char* name, int value) {
    GPP_REQUIRE(name, GPP_ERR_INVALID, "debug_set_option: null name");
    static const char* const names[DBG_COUNT] = {"gf_timing", "tc_timing", "fe_timing", "no_pdl", "gf_mode", "pair_ablate",
                                                  "stage_mode", "lanes"};
    for (int i = 0; i < DBG_COUNT; ++i)
        if (strcmp(name, names[i]) == 0) {
            g_debug_options[i] = value;
            return GPP_OK;
        }
    set_error("debug_set_option: unknown option '%s'", name);
    return GPP_ERR_INVALID;
}

extern "C" int gpp_planner_set_feature_mode(gpp_planner* p, int mode) {
    GPP_REQUIRE(p && mode >= 0 && mode <= 3, GPP_ERR_INVALID, "planner_set_feature_mode: mode must be 0, 1, 2 or 3");
    p->fe_mode = mode;
    return GPP_OK;
}

extern "C" int gpp_planner_set_profiling(gpp_planner* p, int enable) {
    GPP_REQUIRE(p, GPP_ERR_INVALID, "planner_set_profiling: null planner");
    p->profiling = enable != 0;
    if (enable && !p->events) p->events = new std::vector<cudaEvent_t>();
    p->events_used = 0;
    return GPP_OK;
}

extern "C" int gpp_planner_get_profile(gpp_planner* p, double* feature_ms, double* graph_filter_ms, int* steps) {
    GPP_REQUIRE(p, GPP_ERR_INVALID, "planner_get_profile: null planner");
    double fe = 0.0, gf = 0.0;
    const size_t n = p->events_used / 3;
    for (size_t i = 0; i < n; ++i) {
        float a = 0.f, b = 0.f;
        GPP_CUDA_OK(cudaEventSynchronize((*p->events)[3 * i + 2]));
        GPP_CUDA_OK(cudaEventElapsedTime(&a, (*p->events)[3 * i], (*p->events)[3 * i + 1]));
        GPP_CUDA_OK(cudaEventElapsedTime(&b, (*p->events)[3 * i + 1], (*p->events)[3 * i + 2]));
        fe += a;
        gf += b;
    }
    if (feature_ms) *feature_ms = fe;
    if (graph_filter_ms) *graph_filter_ms = gf;
    if (steps) *steps = (int)n;
    p->events_used = 0;
    return GPP_OK;
}

static cudaEvent_t next_event(gpp_planner* p) {
    if (p->events_used == p->events->size()) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
        p->events->push_back(e);
    }
    return (*p->events)[p->events_used++];
}

// Every entry point runs on the handle's device, whatever device the calling thread had current.
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() {
        if (switched) cudaSetDevice(prev);
    }
};

// The handle's scratch (feature workspace, split-filter tickets / partial logits, weight arena) is shared by all
// calls; calls on ONE stream are ordered by the stream.  When the stream changes, the new stream waits for
// everything submitted so far on the previous one (recorded lazily, so the steady state pays nothing).
static int order_after_previous_stream(gpp_planner* p, cudaStream_t st) {
    if (p->last_stream_valid && p->last_stream != st) {
        if (!p->order_event) GPP_CUDA_OK(cudaEventCreateWithFlags(&p->order_event, cudaEventDisableTiming));
        GPP_CUDA_OK(cudaEventRecord(p->order_event, p->last_stream));
        GPP_CUDA_OK(cudaStreamWaitEvent(st, p->order_event, 0));
    }
    p->last_stream = st;
    p->last_stream_valid = true;
    return GPP_OK;
}

extern "C" int gpp_planner_set_weights(gpp_planner* p, const gpp_planner_weights* w, int on_device,
                                       void* stream) {
    GPP_REQUIRE(p && w, GPP_ERR_INVALID, "planner_set_weights: null pointer");
    DeviceGuard guard(p->device);
    cudaStream_t st = on_device ? reinterpret_cast<cudaStream_t>(stream) : p->stream;
    {   // outstanding forwards on another stream still read the arena
        int rc0 = order_after_previous_stream(p, st);
        if (rc0) return rc0;
    }
    for (int l = 0; l < kLanes - 1; ++l)      // batches in flight on the other lanes read the arena
        if (p->lane_stream[l]) GPP_CUDA_OK(cudaStreamSynchronize(p->lane_stream[l]));
    gpp_planner_weights d = *w;
    const int K = p->K;
    if (!on_device) {
        // stage every host array into one device block, then run the same re-layout kernels
        size_t total = 0;
        for (int l = 0; l < 5; ++l) total += (size_t)kConvC[l] * 9 * kConvC[l + 1] + 5 * (size_t)kConvC[l + 1];
        total += 128 * 128 + 128 + (size_t)K * 128 * 128 + 128 + 5 * 128 + 5;
        if (p->raw_floats < total) {
            cudaFree(p->raw);
            p->raw = nullptr;
            GPP_CUDA_OK(cudaMalloc(&p->raw, sizeof(float) * total));
            p->raw_floats = total;
        }
        float* cur = p->raw;
        auto up = [&](const float*& ptr, size_t n) -> cudaError_t {
            cudaError_t e = cudaMemcpyAsync(cur, ptr, sizeof(float) * n, cudaMemcpyHostToDevice, st);
            ptr = cur;
            cur += n;
            return e;
        };
        for (int l = 0; l < 5; ++l) {
            const size_t c = kConvC[l + 1];
            GPP_CUDA_OK(up(d.conv_w[l], (size_t)kConvC[l] * 9 * c));
            GPP_CUDA_OK(up(d.conv_b[l], c));
            GPP_CUDA_OK(up(d.bn_w[l], c));
            GPP_CUDA_OK(up(d.bn_b[l], c));
            GPP_CUDA_OK(up(d.bn_mean[l], c));
            GPP_CUDA_OK(up(d.bn_var[l], c));
        }
        GPP_CUDA_OK(up(d.compress_w, 128 * 128));
        GPP_CUDA_OK(up(d.compress_b, 128));
        GPP_CUDA_OK(up(d.gf_w, (size_t)K * 128 * 128));
        GPP_CUDA_OK(up(d.gf_b, 128));
        GPP_CUDA_OK(up(d.action_w, 5 * 128));
        GPP_CUDA_OK(up(d.action_b, 5));
    }
    float* A = p->arena;
    for (int l = 0; l < 5; ++l) {
        // [Cout][Cin*9] -> [Cin*9][Cout]
        int rc = launch_transpose_taps(d.conv_w[l], A + p->off_w[l], kConvC[l + 1], kConvC[l] * 9, st);
        if (rc) return rc;
        const int C = kConvC[l + 1];
        fold_bn_kernel<<<(C + 127) / 128, 128, 0, st>>>(d.conv_b[l], d.bn_w[l], d.bn_b[l], d.bn_mean[l],
                                                         d.bn_var[l], A + p->off_sc[l], A + p->off_sh[l], C);
        GPP_LAUNCH_CHECK();
    }
    for (int l = 0; l < 6; ++l) {
        int rcf = launch_prep_feature_tc(l < 5 ? d.conv_w[l] : d.compress_w, A + p->off_fimg[l], l, st);
        if (rcf) return rcf;
    }
    int rc = launch_transpose_taps(d.compress_w, A + p->off_w[5], 128, 128, st);
    if (rc) return rc;
    GPP_CUDA_OK(cudaMemcpyAsync(A + p->off_b5, d.compress_b, sizeof(float) * 128, cudaMemcpyDeviceToDevice, st));
    {
        const float* scp[5];
        const float* shp[5];
        for (int l = 0; l < 5; ++l) { scp[l] = A + p->off_sc[l]; shp[l] = A + p->off_sh[l]; }
        rc = launch_prep_feature_mma(d.conv_w, d.compress_w, scp, shp, A + p->off_b5, A + p->off_fmma, st);
        if (rc) return rc;
    }
    rc = launch_transpose_taps(d.gf_w, A + p->off_gfw, 128, K * 128, st);
    if (rc) return rc;
    rc = launch_split_taps(A + p->off_gfw, A + p->off_gfws, K * 128, st);
    p->pdl_ok = false;
    for (int l = 0; l < kLanes - 1; ++l) p->lane_pdl_ok[l] = false;
    if (rc) return rc;
    rc = launch_prep_umma_taps(d.gf_w, A + p->off_gfimg, K, st);
    if (rc) return rc;
    if (K <= 3) {
        rc = launch_prep_pair_taps(d.gf_w, A + p->off_gfpair, K, st);
        if (rc) return rc;
        rc = launch_prep_gf_small(d.gf_w, A + p->off_gfsmall, K, st);
        if (rc) return rc;
    }
    GPP_CUDA_OK(cudaMemcpyAsync(A + p->off_b5, d.compress_b, sizeof(float) * 128, cudaMemcpyDeviceToDevice, st));
    GPP_CUDA_OK(cudaMemcpyAsync(A + p->off_gfb, d.gf_b, sizeof(float) * 128, cudaMemcpyDeviceToDevice, st));
    GPP_CUDA_OK(cudaMemcpyAsync(A + p->off_wa, d.action_w, sizeof(float) * 5 * 128, cudaMemcpyDeviceToDevice, st));
    GPP_CUDA_OK(cudaMemcpyAsync(A + p->off_ba, d.action_b, sizeof(float) * 5, cudaMemcpyDeviceToDevice, st));
    // host copy of the 5 x 128 action MLP (kernel parameters of the CTA-pair filter kernel); weights change rarely
    if (on_device) {
        GPP_CUDA_OK(cudaMemcpyAsync(p->wa_host, d.action_w, sizeof(float) * 5 * 128, cudaMemcpyDeviceToHost, st));
        GPP_CUDA_OK(cudaMemcpyAsync(p->wa_host + 640, d.action_b, sizeof(float) * 5, cudaMemcpyDeviceToHost, st));
        GPP_CUDA_OK(cudaStreamSynchronize(st));
    } else {
        memcpy(p->wa_host, w->action_w, sizeof(float) * 5 * 128);
        memcpy(p->wa_host + 640, w->action_b, sizeof(float) * 5);
        GPP_CUDA_OK(cudaStreamSynchronize(st));
    }
    p->weights_set = true;
    return GPP_OK;
}

// Growing a workspace: stream-ordered free + allocation on the launching stream (the callers have already ordered
// `st` after any other stream that used the handle), so no device-wide synchronisation on the step path.
static int ensure_feat(gpp_planner* p, size_t rows, cudaStream_t st) {
    if (p->feat_rows >= rows) return GPP_OK;
    if (p->feat) GPP_CUDA_OK(cudaFreeAsync(p->feat, st));
    p->feat = nullptr;
    p->feat_rows = 0;
    GPP_CUDA_OK(cudaMallocAsync(&p->feat, sizeof(float) * 128 * rows, st));
    p->feat_rows = rows;
    return GPP_OK;
}

static int ensure_gf_scratch(gpp_planner* p, size_t rows, cudaStream_t st) {
    if (p->gf_lpart_rows >= rows) return GPP_OK;
    if (p->gf_lpart) GPP_CUDA_OK(cudaFreeAsync(p->gf_lpart, st));
    p->gf_lpart = nullptr;
    p->gf_lpart_rows = 0;
    const size_t floats = (size_t)(2 * 5 + 1) * rows;
    GPP_CUDA_OK(cudaMallocAsync(&p->gf_lpart, sizeof(float) * floats, st));
    GPP_CUDA_OK(cudaMemsetAsync(p->gf_lpart, 0, sizeof(float) * floats, st));  // tickets start (and are left) at zero
    p->gf_lpart_rows = rows;
    return GPP_OK;
}

// x / S / logits may be device memory or pinned host memory mapped into the device address space
// (zero-copy); `allow_bulk` = 0 keeps the filter kernel off the bulk-copy engine for host-mapped S.
struct LaneGuard {       // lane l > 0: the handle's scratch fields point at that lane's buffers inside the call
    gpp_planner* p;
    int l;
    void swap_in_out() {
        std::swap(p->feat, p->lane_feat[l]); std::swap(p->feat_rows, p->lane_feat_rows[l]);
        std::swap(p->gf_lpart, p->lane_lpart[l]); std::swap(p->gf_lpart_rows, p->lane_lpart_rows[l]);
        std::swap(p->pdl_ok, p->lane_pdl_ok[l]);
    }
    LaneGuard(gpp_planner* pl, int lane) : p(pl), l(lane - 1) { if (l >= 0) swap_in_out(); }
    ~LaneGuard() { if (l >= 0) swap_in_out(); }
};

static int planner_forward_impl(gpp_planner* p, const float* x, const void* S, int s_is_f64,
                                float* logits, float* features_out, int B, int N, int allow_bulk,
                                cudaStream_t st, int lane = 0) {
    const size_t rows = (size_t)B * N;
    LaneGuard lane_guard(p, lane);
    if (lane == 0) {       // the other lanes' scratch is only ever used on their own streams
        int rc0 = order_after_previous_stream(p, st);
        if (rc0) return rc0;
    }
    float* feat = features_out;
    if (!feat) {
        int rc = ensure_feat(p, rows, st);
        if (rc) return rc;
        feat = p->feat;
    }
    const float* A = p->arena;
    FeArgs fa;
    fa.x = x; fa.feat = feat; fa.total_agents = (int)rows; fa.apt = 0; fa.num_tiles = 0; fa.timing = nullptr;
    // programmatic dependent launch: each kernel's prologue (barriers, filter prefetch) overlaps the tail of the
    // kernel before it; not for the first forward after the weights changed (the prologue reads them)
    // ... and not on the multi-lane pipelined host path: a dependent kernel launched early parks its CTAs (and their shared
    // memory) on the SMs the other lane's kernel should be using
    const int pdl = (!debug_option(DBG_NO_PDL) && p->pdl_ok && !p->profiling && !p->lanes_active) ? 1 : 0;
    fa.pdl = pdl;
    fa.w0t = A + p->off_w[0]; fa.w1t = A + p->off_w[1]; fa.w2t = A + p->off_w[2];
    fa.w3t = A + p->off_w[3]; fa.w4t = A + p->off_w[4]; fa.w5t = A + p->off_w[5];
    for (int l = 0; l < 5; ++l) { fa.sc[l] = A + p->off_sc[l]; fa.sh[l] = A + p->off_sh[l]; }
    fa.b5 = A + p->off_b5;
    const bool prof = p->profiling && p->events && p->events_used + 3 <= 3 * 8192;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr;
    if (prof) {
        e0 = next_event(p); e1 = next_event(p); e2 = next_event(p);
        GPP_REQUIRE(e0 && e1 && e2, GPP_ERR_CUDA, "planner_forward: cudaEventCreate failed");
        GPP_CUDA_OK(cudaEventRecord(e0, st));
    }
    int rc;
    // auto = the im2col-free fp16-split wgmma kernel from 448 agents; small batches (the batch-1 rollout step) stay on the
    // CUDA cores.  Measured on an H100 SXM (400 W power limit): one launch of 640 agents takes 46-53 us on the CUDA cores
    // and 53-58 us in the wgmma kernel, but the wgmma kernel holds one tile of 8 agents per CTA (80 CTAs), leaving SMs
    // to the other batches in flight: bench.py's pipelined value was 14.1-17.0 M agent-steps/s with it against
    // 14.3-14.4 M with the CUDA-core kernel (alternating runs); at 4,100 agents the wgmma kernel also wins a single
    // launch (210 vs 232 us).  The 3xTF32 implicit-GEMM kernel runs on request only.
    if (p->fe_mode == 3 || (p->fe_mode == 0 && rows >= 448)) {
        rc = launch_feature_mma_kernel(fa, A + p->off_fmma, allow_bulk, st);
    } else if (p->fe_mode == 2) {
        const float* imgs[6];
        for (int l = 0; l < 6; ++l) imgs[l] = A + p->off_fimg[l];
        rc = launch_feature_tc_kernel(fa, imgs, st);
    } else {
        rc = launch_feature_kernel(fa, st);
    }
    if (rc) return rc;
    if (prof) GPP_CUDA_OK(cudaEventRecord(e1, st));
    const bool tc_fits = gf_tc_tile_samples(N, p->K) > 0;
    GPP_REQUIRE(p->gf_mode != 2 || tc_fits, GPP_ERR_UNSUPPORTED,
                "planner_forward: tensor-core graph filter requested but N=%d K=%d does not fit its tile", N, p->K);
    const bool pair_fits = gf_pair_supported(N, p->K);
    GPP_REQUIRE(p->gf_mode != 3 || pair_fits, GPP_ERR_UNSUPPORTED,
                "planner_forward: CTA-pair graph filter requested but N=%d K=%d is outside its envelope", N, p->K);
    const bool use_pair = pair_fits && (p->gf_mode == 3 || (p->gf_mode == 0 && rows >= 4096));
    const bool use_tc = !use_pair && tc_fits && (p->gf_mode == 2 || (p->gf_mode == 0 && rows >= 4096));
    // small batches at N = 10 (the benchmark configuration, rollout steps): 2 CTAs per 6 samples on the tensor core
    const bool use_small = !use_pair && p->gf_mode == 0 && gf_small_supported(N, p->K) && !debug_option(DBG_GF_MODE);
    if (use_small) {
        rc = launch_gf_forward_small(feat, S, s_is_f64, A + p->off_gfsmall, A + p->off_gfb, A + p->off_wa, A + p->off_ba,
                                     logits, B, p->K, pdl, st);
    } else if (use_pair)
        rc = launch_gf_forward_pair(feat, S, s_is_f64, A + p->off_gfpair, A + p->off_gfb, nullptr, p->wa_host,
                                    p->wa_host + 640, logits, B, N, p->K, 1, st);
    else if (use_tc)
        rc = launch_gf_forward_tc(feat, S, s_is_f64, A + p->off_gfimg, A + p->off_gfb, nullptr, A + p->off_wa,
                                  A + p->off_ba, logits, B, N, p->K, 1, allow_bulk, st);
    else {
        rc = ensure_gf_scratch(p, rows, st);
        if (rc) return rc;
        rc = launch_gf_forward_fast(feat, S, s_is_f64, A + p->off_gfw, A + p->off_gfb, nullptr,
                                    A + p->off_wa, A + p->off_ba, logits, B, N, p->K, GPP_NODE_MAJOR,
                                    GPP_NODE_MAJOR, 1, allow_bulk, p->gf_lpart,
                                    reinterpret_cast<unsigned int*>(p->gf_lpart + 10 * p->gf_lpart_rows),
                                    A + p->off_gfws, pdl, st);
    }
    if (rc) return rc;
    if (prof) GPP_CUDA_OK(cudaEventRecord(e2, st));
    p->pdl_ok = true;
    return GPP_OK;
}

extern "C" int gpp_planner_forward(gpp_planner* p, const float* x, const void* S, int s_is_f64,
                                   float* logits, float* features_out, int B, int N, void* stream) {
    GPP_REQUIRE(p && x && S && logits, GPP_ERR_INVALID, "planner_forward: null pointer");
    DeviceGuard guard(p->device);
    GPP_REQUIRE((reinterpret_cast<uintptr_t>(features_out) & 15) == 0, GPP_ERR_INVALID,
                "planner_forward: features_out must be 16-byte aligned");
    GPP_REQUIRE(p->weights_set, GPP_ERR_INVALID, "planner_forward: gpp_planner_set_weights not called");
    GPP_REQUIRE(B >= 0 && N >= 1, GPP_ERR_INVALID, "planner_forward: bad sizes B=%d N=%d", B, N);
    GPP_REQUIRE(N <= 64, GPP_ERR_UNSUPPORTED, "planner_forward: N=%d > 64 agents is outside the fused kernel's tile", N);
    if (B == 0) return GPP_OK;
    return planner_forward_impl(p, x, S, s_is_f64, logits, features_out, B, N, 1,
                                reinterpret_cast<cudaStream_t>(stream));
}

// Returns the device alias of a pinned (page-locked, device-mapped) host pointer, or null for
// pageable host memory.
static void* mapped_alias(const void* host_ptr) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, host_ptr) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    if (at.type == cudaMemoryTypeHost && at.devicePointer) return at.devicePointer;
    return nullptr;
}
// The per-step calls of a rollout cycle through a handful of pinned buffers: remember their device aliases
// (a pinned allocation keeps its alias for its lifetime; a freed one that comes back is simply looked up again
// after it falls out of the 16 most recent entries or fails the cheap pointer check below).
static void* mapped_alias_cached(gpp_planner* p, const void* host_ptr) {
    for (int i = 0; i < 16; ++i)
        if (p->alias_host[i] == host_ptr && host_ptr) return p->alias_dev[i];
    void* d = mapped_alias(host_ptr);
    if (d) {
        const int i = (int)(p->alias_next++ & 15);
        p->alias_host[i] = host_ptr;
        p->alias_dev[i] = d;
    }
    return d;
}

// kLanes compute lanes (stream + feature workspace + filter scratch each), tickets rotate over them: the batches are
// independent, so the feature kernel of ticket t+1 (80 of the SMs at the benchmark size) runs next to the kernels of
// the tickets before it instead of behind them.  `ready`: the inputs are complete once this event has fired.
static int enqueue_on_lane(gpp_planner* p, const float* x, const void* S, int s_is_f64, float* logits, int B, int N,
                           cudaEvent_t ready, unsigned long long* ticket) {
    const unsigned long long t = p->next_ticket;
    cudaEvent_t& ev = p->tickets[t % 16];
    if (!ev) GPP_CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    const int nlanes = debug_option(DBG_LANES) >= 1 && debug_option(DBG_LANES) <= kLanes ? debug_option(DBG_LANES) : kLanes;
    const int lane = (int)(t % (unsigned long long)nlanes);
    if (lane && !p->lane_stream[lane - 1])
        GPP_CUDA_OK(cudaStreamCreateWithFlags(&p->lane_stream[lane - 1], cudaStreamNonBlocking));
    cudaStream_t cst = lane ? p->lane_stream[lane - 1] : p->stream;
    GPP_CUDA_OK(cudaStreamWaitEvent(cst, ready, 0));
    p->lanes_active = true;
    int rc = planner_forward_impl(p, x, S, s_is_f64, logits, nullptr, B, N, 1, cst, lane);
    p->lanes_active = false;
    if (rc) return rc;
    GPP_CUDA_OK(cudaEventRecord(ev, cst));
    p->next_ticket = t + 1;
    *ticket = t;
    return GPP_OK;
}

extern "C" int gpp_planner_forward_host_async(gpp_planner* p, const float* x_host, const void* S_host,
                                              int s_is_f64, float* logits_host, int B, int N,
                                              unsigned long long* ticket) {
    GPP_REQUIRE(p && x_host && S_host && logits_host && ticket, GPP_ERR_INVALID, "planner_forward_host_async: null pointer");
    DeviceGuard guard(p->device);
    GPP_REQUIRE(p->weights_set, GPP_ERR_INVALID, "planner_forward_host_async: gpp_planner_set_weights not called");
    GPP_REQUIRE(B >= 1 && N >= 1 && N <= 64, GPP_ERR_INVALID, "planner_forward_host_async: bad sizes B=%d N=%d", B, N);
    void* mx = mapped_alias_cached(p, x_host);
    void* mS = mapped_alias_cached(p, S_host);
    void* ml = mapped_alias_cached(p, logits_host);
    GPP_REQUIRE(mx && mS && ml, GPP_ERR_INVALID,
                "planner_forward_host_async: buffers must be pinned (page-locked) host memory");
    GPP_REQUIRE((reinterpret_cast<uintptr_t>(mx) & 15u) == 0 && (reinterpret_cast<uintptr_t>(mS) & 15u) == 0,
                GPP_ERR_INVALID, "planner_forward_host_async: host buffers must be 16-byte aligned");
    const unsigned long long t = p->next_ticket;
    // Pipelined path: the inputs of this step are moved by the copy engine on a copy
    // stream into one of kStageSlots device slots while the kernels of the previous steps run on the compute streams (a kernel that reads its
    // input straight over PCIe cannot overlap that read with its own compute); the logits are still
    // written straight into the pinned host buffer.  Slot reuse waits for the step kStageSlots tickets back.
    const int slot = (int)(t % kStageSlots);
    const size_t nx = (size_t)B * N * IN_PIX;
    const size_t sb = (size_t)B * N * N * (s_is_f64 ? 8 : 4);
    if (!p->copy_stream) GPP_CUDA_OK(cudaStreamCreateWithFlags(&p->copy_stream, cudaStreamNonBlocking));
    if (!p->copied[slot]) GPP_CUDA_OK(cudaEventCreateWithFlags(&p->copied[slot], cudaEventDisableTiming));
    if (p->a_x_floats[slot] < nx || p->a_S_bytes[slot] < sb) {
        GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
        for (int l = 0; l < kLanes - 1; ++l)
            if (p->lane_stream[l]) GPP_CUDA_OK(cudaStreamSynchronize(p->lane_stream[l]));
        GPP_CUDA_OK(cudaStreamSynchronize(p->copy_stream));
        if (p->a_x_floats[slot] < nx) {
            cudaFree(p->a_x[slot]); p->a_x[slot] = nullptr; p->a_x_floats[slot] = 0;
            GPP_CUDA_OK(cudaMalloc(&p->a_x[slot], sizeof(float) * nx));
            p->a_x_floats[slot] = nx;
        }
        if (p->a_S_bytes[slot] < sb) {
            cudaFree(p->a_S[slot]); p->a_S[slot] = nullptr; p->a_S_bytes[slot] = 0;
            GPP_CUDA_OK(cudaMalloc(&p->a_S[slot], sb));
            p->a_S_bytes[slot] = sb;
        }
    }
    if (t >= (unsigned long long)kStageSlots)
        GPP_CUDA_OK(cudaStreamWaitEvent(p->copy_stream, p->tickets[(t - kStageSlots) % 16], 0));
    {
        const size_t xb = sizeof(float) * nx;
        // The copy engine moves the step's inputs; the staging kernel (a few CTAs pulling pinned memory with 16-byte loads) needs 5+ batches in
        // flight to match it and is kept behind the "stage_mode" debug option for the probe.
        if (debug_option(DBG_STAGE_MODE) == 0) {
            GPP_CUDA_OK(cudaMemcpyAsync(p->a_x[slot], x_host, xb, cudaMemcpyHostToDevice, p->copy_stream));
            GPP_CUDA_OK(cudaMemcpyAsync(p->a_S[slot], S_host, sb, cudaMemcpyHostToDevice, p->copy_stream));
        } else {
            StagePair sp;
            sp.src[0] = reinterpret_cast<const uint4*>(mx); sp.dst[0] = reinterpret_cast<uint4*>(p->a_x[slot]);
            sp.n16[0] = xb / 16; sp.tail[0] = (int)(xb % 16);
            sp.src[1] = reinterpret_cast<const uint4*>(mS); sp.dst[1] = reinterpret_cast<uint4*>(p->a_S[slot]);
            sp.n16[1] = sb / 16; sp.tail[1] = (int)(sb % 16);
            stage_h2d_pair_kernel<<<16 + 1, 256, 0, p->copy_stream>>>(sp);
            GPP_LAUNCH_CHECK();
        }
    }
    GPP_CUDA_OK(cudaEventRecord(p->copied[slot], p->copy_stream));
    return enqueue_on_lane(p, p->a_x[slot], p->a_S[slot], s_is_f64, reinterpret_cast<float*>(ml), B, N, p->copied[slot], ticket);
}

extern "C" int gpp_planner_forward_async(gpp_planner* p, const float* x, const void* S, int s_is_f64, float* logits,
                                         int B, int N, void* stream, unsigned long long* ticket) {
    GPP_REQUIRE(p && x && S && logits && ticket, GPP_ERR_INVALID, "planner_forward_async: null pointer");
    DeviceGuard guard(p->device);
    GPP_REQUIRE(p->weights_set, GPP_ERR_INVALID, "planner_forward_async: gpp_planner_set_weights not called");
    GPP_REQUIRE(B >= 1 && N >= 1 && N <= 64, GPP_ERR_INVALID, "planner_forward_async: bad sizes B=%d N=%d", B, N);
    cudaEvent_t& rd = p->ready[p->next_ticket % 16];
    if (!rd) GPP_CUDA_OK(cudaEventCreateWithFlags(&rd, cudaEventDisableTiming));
    GPP_CUDA_OK(cudaEventRecord(rd, reinterpret_cast<cudaStream_t>(stream)));     // x and S are ready behind this point
    return enqueue_on_lane(p, x, S, s_is_f64, logits, B, N, rd, ticket);
}

extern "C" int gpp_planner_join(gpp_planner* p, unsigned long long ticket, void* stream) {
    GPP_REQUIRE(p, GPP_ERR_INVALID, "planner_join: null planner");
    DeviceGuard guard(p->device);
    GPP_REQUIRE(ticket < p->next_ticket && ticket + 16 >= p->next_ticket, GPP_ERR_INVALID,
                "planner_join: ticket %llu is not among the 16 most recent calls", ticket);
    GPP_CUDA_OK(cudaStreamWaitEvent(reinterpret_cast<cudaStream_t>(stream), p->tickets[ticket % 16], 0));
    return GPP_OK;
}

extern "C" int gpp_planner_wait(gpp_planner* p, unsigned long long ticket) {
    GPP_REQUIRE(p, GPP_ERR_INVALID, "planner_wait: null planner");
    DeviceGuard guard(p->device);
    GPP_REQUIRE(ticket < p->next_ticket && ticket + 16 >= p->next_ticket, GPP_ERR_INVALID,
                "planner_wait: ticket %llu is not among the 16 most recent calls", ticket);
    GPP_CUDA_OK(cudaEventSynchronize(p->tickets[ticket % 16]));
    return GPP_OK;
}

extern "C" int gpp_planner_forward_host(gpp_planner* p, const float* x_host, const void* S_host,
                                        int s_is_f64, float* logits_host, int B, int N) {
    GPP_REQUIRE(p && x_host && S_host && logits_host, GPP_ERR_INVALID, "planner_forward_host: null pointer");
    DeviceGuard guard(p->device);
    GPP_REQUIRE(p->weights_set, GPP_ERR_INVALID, "planner_forward_host: gpp_planner_set_weights not called");
    GPP_REQUIRE(B >= 0 && N >= 1, GPP_ERR_INVALID, "planner_forward_host: bad sizes B=%d N=%d", B, N);
    GPP_REQUIRE(N <= 64, GPP_ERR_UNSUPPORTED, "planner_forward_host: N=%d > 64 agents", N);
    if (B == 0) return GPP_OK;
    const size_t nx = (size_t)B * N * IN_PIX;
    const size_t sb = (size_t)B * N * N * (s_is_f64 ? 8 : 4);
    const size_t nl = (size_t)B * N * 5;
    // Zero-copy path: with pinned buffers the kernels read x / S straight from host memory over
    // PCIe and write the logits straight back -- no staging copies, no extra launches.  The FOV
    // tensor is read exactly once (by the staging loop of the feature kernel), so a separate
    // H2D copy would move the same bytes and add its own launch + completion latency.
    void* mx = mapped_alias(x_host);
    void* mS = mapped_alias(S_host);
    void* ml = mapped_alias(logits_host);
    if (mx && mS && ml) {
        int rc = planner_forward_impl(p, reinterpret_cast<const float*>(mx), mS, s_is_f64,
                                      reinterpret_cast<float*>(ml), nullptr, B, N, 0, p->stream);
        if (rc) return rc;
        GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
        return GPP_OK;
    }
    // Pageable host memory: staged copies on the planner's stream.
    if (p->d_x_floats < nx) {
        GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
        cudaFree(p->d_x); p->d_x = nullptr; p->d_x_floats = 0;
        GPP_CUDA_OK(cudaMalloc(&p->d_x, sizeof(float) * nx));
        p->d_x_floats = nx;
    }
    if (p->d_S_bytes < sb) {
        GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
        cudaFree(p->d_S); p->d_S = nullptr; p->d_S_bytes = 0;
        GPP_CUDA_OK(cudaMalloc(&p->d_S, sb));
        p->d_S_bytes = sb;
    }
    if (p->d_logits_floats < nl) {
        GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
        cudaFree(p->d_logits); p->d_logits = nullptr; p->d_logits_floats = 0;
        GPP_CUDA_OK(cudaMalloc(&p->d_logits, sizeof(float) * nl));
        p->d_logits_floats = nl;
    }
    GPP_CUDA_OK(cudaMemcpyAsync(p->d_x, x_host, sizeof(float) * nx, cudaMemcpyHostToDevice, p->stream));
    GPP_CUDA_OK(cudaMemcpyAsync(p->d_S, S_host, sb, cudaMemcpyHostToDevice, p->stream));
    int rc = planner_forward_impl(p, p->d_x, p->d_S, s_is_f64, p->d_logits, nullptr, B, N, 1, p->stream);
    if (rc) return rc;
    GPP_CUDA_OK(cudaMemcpyAsync(logits_host, p->d_logits, sizeof(float) * nl, cudaMemcpyDeviceToHost, p->stream));
    GPP_CUDA_OK(cudaStreamSynchronize(p->stream));
    return GPP_OK;
}
