// Host side of libsmap_b200: handle, weight folding/repack, execution plan, C ABI (include/smap_b200.h).
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <nvtx3/nvToolsExt.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/smap_b200.h"
#include "../../include/smap_b200_debug.h"
#include "assoc.h"
#include "conv_tc.cuh"
#include "elementwise.h"
#include "preprocess.h"
#include "refine.h"

using namespace smapb;

namespace {

// ------------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------------
thread_local std::string g_create_error = "";

// Process-wide tile-shape table: layer geometry -> (BLOCK_N, CTA-group size).  Filled from the committed table
// (smapb_set_tile_table) and, for geometries it does not cover, by the autotuner.  Being process-wide, every handle of a
// process runs a given layer with the same tile shape; across processes the committed table (or a broadcast of rank 0's
// table, smap_b200.dist.sync_tile_table) gives the same guarantee.
std::mutex g_tiles_mu;
std::map<std::string, std::pair<int, int>> g_tiles;

inline uint16_t f32_to_bf16_rn(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
    const uint32_t lsb = (u >> 16) & 1u;
    u += 0x7fffu + lsb;
    return (uint16_t)(u >> 16);
}
inline float bf16_to_f32(uint16_t b) {
    uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
inline uint16_t f32_to_f16_rn(float f) { return __half_as_ushort(__float2half_rn(f)); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// split-bf16 NHWC activation tensor: plane 0 = hi, plane 1 = lo
struct Act {
    __nv_bfloat16* ptr = nullptr;
    int N = 0, H = 0, W = 0, C = 0;
    long long plane() const { return (long long)N * H * W * C; }
};
struct ActF32 {
    float* ptr = nullptr;
    int N = 0, H = 0, W = 0, C = 0;
};

struct ConvLayer {
    std::string name;
    int Cin = 0, Cout = 0, Cout_pad = 0, k = 1, stride = 1, pad = 0, relu = 0;
    int Cin2 = 0, stride2 = 1;  // K-concatenated second 1x1 input (weights hold Cin + Cin2 columns)
    bool stem_s2d = false;      // space-to-depth stem: 4x1 taps over a sliding 4-pixel window view (see build_plan)
    __nv_bfloat16* w_dev = nullptr;  // [T][taps][Cout_pad][Cin]
    float* bias_dev = nullptr;       // [Cout_pad]
};

enum OpKind { OP_STEM, OP_S2D, OP_MAXPOOL, OP_CONV, OP_UPADD, OP_HEADMERGE, OP_TAPSUM };
struct Op {
    OpKind kind;
    // conv
    ConvParams cp;
    int block_n = 0;
    int cg = 1;  // tile-table variant (1: one CTA per tile, the only one built)
    double flops = 0;
    // generic tensors
    Act a, b, out;
    ActF32 f4, f3, f2;
    int cout = 0;  // head merge real channel count
    int which_out = 0;  // 0 hm2d, 1 detd, 2 rootd
    const float* bias = nullptr;  // tap-sum bias
    // two-stream execution: side-branch ops (skip convs, heads) run on stream 1 and overlap the main chain
    int stream = 0;
    std::vector<int> waits;  // indices of producer ops on the OTHER stream this op must wait for
    bool record = false;     // some op on the other stream consumes this op's output
    cudaEvent_t ev = nullptr;
    std::string name;  // reference unit name (NVTX range, profiles)
    // debug descriptions (smapb_debug_checksums): the tensors the op reads, in the order PlanBuilder::wire received them
    // (conv: in, res, p1, p2, in2, up; null = role absent), and the output shape N, H, W, C of a conv
    std::vector<const void*> inputs;
    int dims[4] = {0, 0, 0, 0};
};

struct Plan {
    int B = 0;
    std::vector<Op> ops;
    std::vector<void*> allocs;
    int n_conv = 0;
    double conv_flops = 0;
    cudaGraphExec_t graph = nullptr;
    std::map<const void*, int> producer;  // tensor -> index of the op that writes it (build time)
    int last_side = -1;
};

}  // namespace

struct smapb_handle {
    int device = 0, max_batch = 0, in_h = 0, in_w = 0, h = 0, w = 0;
    int sm_count = 132;
    int sm_reserve = 0;  // SMs the persistent conv grids leave to concurrent kernels
    std::string err;
    int64_t launches = 0;
    // weights
    std::map<std::string, std::vector<float>> raw;
    std::map<std::string, std::vector<int64_t>> raw_shape;
    std::map<std::string, ConvLayer> layers;
    float* stem_w = nullptr;  // [147][64]
    ConvLayer stem_tc;        // space-to-depth tensor-core stem (4 ky-blocks x 64 k)
    int stem_tc_ok = -1;      // -1 untested, 0 overlapped TMA view rejected (CUDA-core stem), 1 in use
    float* stem_b = nullptr;
    int nterms = 3;  // MMA terms (3 = bf16x3, 1 = bf16 or fp16)
    int planes = 2;  // activation planes (2 or 1)
    bool f16 = false;  // element format of weights and activations: fp16 (SMAPB_PREC_FP16) instead of bf16
    unsigned long long* sat_dev = nullptr;  // fp16: activation elements clamped to +-65504 (smapb_saturation_count)
    bool finalized = false;
    std::map<int, std::unique_ptr<Plan>> plans;
    // association workspace (sized for max_batch)
    float* peaks = nullptr;
    float* scores = nullptr;
    float* bodies = nullptr;
    int* counts = nullptr;
    uint32_t* nms_masks = nullptr;  // one ballot bit per pixel of the key-point planes
    // whole-path workspace
    float* imgs_dev = nullptr;
    float* imgs_flip = nullptr;
    float* hm = nullptr;
    float* hm_flip = nullptr;
    float* detd = nullptr;
    float* rootd = nullptr;
    float* scratch_detd = nullptr;
    float* scratch_rootd = nullptr;
    double* scales_dev = nullptr;
    smapb_record* records_dev = nullptr;
    bool use_pdl = getenv("SMAPB_PDL") != nullptr;  // programmatic dependent launch between conv kernels
    // host-facing pipeline (smapb_submit_host / smapb_wait): two slots, H2D of slot s+1 overlaps the compute of slot s
    struct Slot {
        float* imgs = nullptr;
        double* scales = nullptr;
        smapb_record* records = nullptr;
        smapb_record* records_all = nullptr;  // [comm_world * max_batch], gathered variant
        cudaEvent_t h2d = nullptr, done = nullptr, rec_ready = nullptr;
        bool used = false;
    } slots[2];
    cudaStream_t copy_stream = nullptr;
    bool autotune = getenv("SMAPB_NO_AUTOTUNE") == nullptr;
    bool two_streams = getenv("SMAPB_ONE_STREAM") == nullptr;  // side branches (heads, skip convs) on a second stream
    cudaStream_t aux_stream = nullptr;  // side branches of the decoder (skip convs, heads) run here
    // Stream used when the caller passes NULL (= the legacy default stream).  It is NON-blocking - a blocking stream would
    // be fenced by every legacy-stream operation of the process (e.g. a collective issued by the host framework) - and is
    // ordered against the legacy stream explicitly with the two bridge events (legacy_enter / legacy_leave).
    cudaStream_t own_stream = nullptr;
    cudaEvent_t bridge_in = nullptr, bridge_out = nullptr;
    struct GraphEntry {
        int B, flip, gather;
        const void* imgs;
        const void* scales;
        cudaGraphExec_t exec;
        uint64_t stamp;  // last use (LRU eviction)
    };
    std::vector<GraphEntry> graphs;  // whole-path CUDA graphs keyed by (B, flip, gather, input pointers)
    uint64_t graph_clock = 0;
    // skeleton-record exchange (SURVEY 8(e)): one ncclAllGather per batch on the compute stream, inside the graph
    void* comm = nullptr;  // ncclComm_t
    bool comm_owned = false;
    int comm_rank = 0, comm_world = 1;
    smapb_record* gather_dev = nullptr;  // [comm_world * max_batch]
    // decoupled exchange (smapb_infer_device_gather_async / smapb_submit_host_gather): the all-gather runs on its own stream
    // behind an event, so a rank's compute stream never waits for its peers
    cudaStream_t gather_stream = nullptr;
    cudaEvent_t rec_ready[2] = {nullptr, nullptr}, gather_done[2] = {nullptr, nullptr};
    smapb_record* rec_buf[2] = {nullptr, nullptr};  // [max_batch] each: the records of the two most recent async calls
    bool gather_used[2] = {false, false};
    int gather_idx = 0;
    double* gt_dist = nullptr;           // [max_batch][127*127] distance matrices of the GT-matching lift
    bool nccl_in_graph = getenv("SMAPB_NCCL_EAGER") == nullptr;
    bool nvtx_ops = getenv("SMAPB_NVTX") != nullptr;  // one NVTX range per plan op (phase ranges are always emitted)
    bool serpentine = getenv("SMAPB_SERPENTINE") != nullptr;
    // pre-processing (SURVEY 8(f) f1): resampling tables per source geometry, staging for host images
    struct PreEntry {
        ResizePlan plan;
        ResizeTablesDev tab{};
        void* buf = nullptr;
    };
    std::map<std::pair<int, int>, PreEntry> pre_cache;
    uint8_t* pre_stage = nullptr;
    size_t pre_stage_bytes = 0;
    // RefineNet (optional post-processing step, SURVEY 8(f) f2)
    std::map<std::string, std::vector<float>> refine_raw;
    float* refine_buf = nullptr;  // folded, transposed weights + biases of the five layers
    RefineWeights refine_w{};
    bool refine_ready = false, refine_on = false;
    std::map<std::pair<int, int>, int> eager_runs;  // (B, flip) -> number of eager executions so far
    // profiling (per-op CUDA events on the launching stream)
    bool profiling = false;
    std::vector<cudaEvent_t> prof_events;
    std::vector<int> prof_kind;          // kind of the op that ended at event i (-1 = interval start)
    std::vector<std::string> prof_desc;  // description of that op
    std::vector<double> prof_flops;
    size_t prof_used = 0;
    // per-launch role counters of the conv kernels inside a profiled (eager) run: SMAPB_ROLES_PLAN=<csv path>
    long long* roles_dev = nullptr;  // [ROLES_CAP][16]
    size_t roles_used = 0;
    std::vector<std::string> roles_desc;
};
constexpr size_t ROLES_CAP = 4096;

namespace {

int fail(smapb_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    return code;
}
#define CK(call)                                                                                          \
    do {                                                                                                  \
        cudaError_t e_ = (call);                                                                          \
        if (e_ != cudaSuccess)                                                                            \
            return fail(h, -10, std::string(#call) + ": " + cudaGetErrorString(e_) + " @" + std::to_string(__LINE__)); \
    } while (0)

// ------------------------------------------------------------------------------------------------
// NCCL, bound at run time (dlopen): libsmap_b200.so has no link-time dependency on it, and inside a PyTorch process
// dlopen("libnccl.so.2") resolves to the instance torch already loaded, so a communicator created by the host framework
// (ProcessGroupNCCL._comm_ptr) and one created here (smapb_comm_create) are served by the same library.
// ------------------------------------------------------------------------------------------------
struct NcclUid {  // ncclUniqueId
    char internal[128];
};
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(NcclUid*) = nullptr;
    int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;  // (ncclComm_t*, nranks, id by value, rank)
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
    std::string err;
};
NcclApi& nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {getenv("SMAPB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) {
            api.err = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "");
            return;
        }
        api.GetUniqueId = (int (*)(NcclUid*))dlsym(api.lib, "ncclGetUniqueId");
        api.CommInitRank = (int (*)(void**, int, NcclUid, int))dlsym(api.lib, "ncclCommInitRank");
        api.CommDestroy = (int (*)(void*))dlsym(api.lib, "ncclCommDestroy");
        api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(api.lib, "ncclAllGather");
        api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
        api.GetVersion = (int (*)(int*))dlsym(api.lib, "ncclGetVersion");
        if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather) {
            api.err = "NCCL library lacks a required symbol";
            api.lib = nullptr;
        }
    });
    return api;
}
int nccl_fail(smapb_handle* h, const char* what, int rc) {
    NcclApi& a = nccl_api();
    return fail(h, -50, std::string(what) + ": " + (a.GetErrorString ? a.GetErrorString(rc) : "NCCL error") + " (" +
                            std::to_string(rc) + ")");
}

// NULL-stream callers (the legacy default stream): order the handle's non-blocking stream after the legacy stream's
// pending work, and - on the way out - the legacy stream after ours, which is what a blocking stream would give them,
// without fencing every other stream of the process.
int legacy_enter(smapb_handle* h) {
    CK(cudaEventRecord(h->bridge_in, cudaStreamLegacy));
    CK(cudaStreamWaitEvent(h->own_stream, h->bridge_in, 0));
    return 0;
}
int legacy_leave(smapb_handle* h) {
    CK(cudaEventRecord(h->bridge_out, h->own_stream));
    CK(cudaStreamWaitEvent(cudaStreamLegacy, h->bridge_out, 0));
    return 0;
}

enum ProfKind { PK_START = -1, PK_CONV = 0, PK_STEM = 1, PK_ELEM = 2, PK_ASSOC = 3, PK_LIFT = 4, PK_COPY = 5 };
void prof_mark(smapb_handle* h, int kind, cudaStream_t st, const char* desc = "", double flops = 0) {
    if (!h->profiling) return;
    if (h->prof_used == h->prof_events.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        h->prof_events.push_back(e);
        h->prof_kind.push_back(0);
        h->prof_desc.emplace_back();
        h->prof_flops.push_back(0);
    }
    cudaEventRecord(h->prof_events[h->prof_used], st);
    h->prof_kind[h->prof_used] = kind;
    h->prof_desc[h->prof_used] = desc;
    h->prof_flops[h->prof_used] = flops;
    h->prof_used++;
}

template <typename T>
int dev_alloc(smapb_handle* h, T** p, size_t count) {
    CK(cudaMalloc((void**)p, count * sizeof(T)));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// tensor maps
// ------------------------------------------------------------------------------------------------
CUtensorMapDataType elem_dtype(const smapb_handle* h) { return h->f16 ? ElemF16::TMA_DTYPE : ElemBF16::TMA_DTYPE; }
int make_act_map(smapb_handle* h, CUtensorMap* m, const __nv_bfloat16* ptr, long long C, long long W, long long H,
                 long long N, int T, long long plane_elems, int box_w, int box_h, int stride, int box_c = 64) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return fail(h, -20, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N, (cuuint64_t)T};
    cuuint64_t strides[4] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2,
                             (cuuint64_t)plane_elems * 2};
    cuuint32_t box[5] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
    cuuint32_t es[5] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1, 1};
    // 64-channel boxes (operands) use 128-byte rows, 32-channel boxes (epilogue tiles) 64-byte rows
    CUresult r = fn(m, elem_dtype(h), 5, (void*)ptr, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, box_c == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled(act) failed: %d  dims=(%lld,%lld,%lld,%lld,%d) box=(64,%d,%d) s=%d",
                 (int)r, C, W, H, N, T, box_w, box_h, stride);
        return fail(h, -21, buf);
    }
    return 0;
}
int make_w_map(smapb_handle* h, CUtensorMap* m, const __nv_bfloat16* ptr, int Cin, int Cout_pad, int taps, int T,
               int block_n) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return fail(h, -20, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)Cout_pad, (cuuint64_t)taps, (cuuint64_t)T};
    cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cout_pad * Cin * 2, (cuuint64_t)taps * Cout_pad * Cin * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)block_n, 1, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(m, elem_dtype(h), 4, (void*)ptr, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(h, -21, "cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// conv launch
// ------------------------------------------------------------------------------------------------
template <int BN, int NT, int RING, class E>
cudaError_t launch_conv_inst2(const ConvParams& cp, int sm_count, cudaStream_t st, bool pdl) {
    using Cfg = ConvCfg<BN, NT, RING>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, NT, RING, E>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    const int units = cp.total_tiles < sm_count ? cp.total_tiles : sm_count;  // persistent CTAs
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(units);
    cfg.blockDim = dim3(384);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    int na = 0;
    if (pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        na++;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, NT, RING, E>, cp);
}
template <int BN, int NT, class E = ElemBF16>
cudaError_t launch_conv_inst(const ConvParams& cp, int sm_count, cudaStream_t st, bool pdl) {
    if (cp.up_mode) return launch_conv_inst2<BN, NT, 2, E>(cp, sm_count, st, pdl);  // fused bilinear residual
    return (cp.has_res + cp.n_post) ? launch_conv_inst2<BN, NT, 1, E>(cp, sm_count, st, pdl)
                                    : launch_conv_inst2<BN, NT, 0, E>(cp, sm_count, st, pdl);
}
cudaError_t launch_conv(const ConvParams& cp, int block_n, int nterms, bool f16, int sm_count, cudaStream_t st, bool pdl) {
#define SMAPB_CASE(BN)                                                                  \
    case BN:                                                                            \
        if (f16) return launch_conv_inst<BN, 1, ElemF16>(cp, sm_count, st, pdl);        \
        return nterms == 3 ? launch_conv_inst<BN, 3>(cp, sm_count, st, pdl)             \
                           : launch_conv_inst<BN, 1>(cp, sm_count, st, pdl);
    switch (block_n) {
        SMAPB_CASE(128)
        SMAPB_CASE(64)
        SMAPB_CASE(32)
    }
#undef SMAPB_CASE
    return cudaErrorInvalidValue;
}

// The tile shapes the kernel is built for: one CTA per 128-row tile (tile-table variant 1) of 32, 64 or 128 columns
bool tile_shape_ok(int bn, int cg) { return cg == 1 && (bn == 32 || bn == 64 || bn == 128); }

// Fill a ConvParams for `layer` applied to `in`, producing (out | out_f32).
int setup_conv(smapb_handle* h, const ConvLayer& L, const Act& in, const Act* res, const Act* post1, const Act* post2,
               const Act* out, const ActF32* outf, int relu, ConvParams* cp, int* block_n_out, double* flops_out,
               const Act* in2 = nullptr, const Act* up = nullptr, int* cg_out = nullptr, int force_bn = 0,
               int force_cg = 0) {
    const int Ho = (in.H + 2 * L.pad - L.k) / L.stride + 1, Wo = (in.W + 2 * L.pad - L.k) / L.stride + 1;
    const int N = in.N;
    if (in.C != L.Cin) return fail(h, -30, "conv " + L.name + ": Cin mismatch");
    if (L.Cin % 64 != 0) return fail(h, -30, "conv " + L.name + ": Cin must be a multiple of 64");
    memset(cp, 0, sizeof(*cp));
    if ((L.Cin2 != 0) != (in2 != nullptr)) return fail(h, -30, "conv " + L.name + ": second input mismatch");
    if (in2 && (in2->C != L.Cin2 || L.k != 1 || L.stride != 1)) return fail(h, -30, "conv " + L.name + ": bad fused pair");
    if (up && (res || post1)) return fail(h, -30, "conv " + L.name + ": up-residual excludes other epilogue inputs");
    const bool flat = (L.k == 1 && L.stride == 1 && (!in2 || L.stride2 == 1) && !up);
    if (!force_bn && getenv("SMAPB_FORCE_TILE")) {  // debug: "bn[,1]" for every layer where it is valid
        int fb = 0, fc = 1;
        if (sscanf(getenv("SMAPB_FORCE_TILE"), "%d,%d", &fb, &fc) >= 1 && tile_shape_ok(fb, fc) && L.Cout_pad % fb == 0)
            force_bn = fb, force_cg = fc;
    }
    int tw, th, tiles_x, tiles_y, nimg;
    int rc;
    if (flat) {
        tw = 128;
        th = 1;
        const long long M = (long long)N * Ho * Wo;
        tiles_x = (int)((M + 127) / 128);
        tiles_y = 1;
        nimg = 1;
        cp->Hout = 1;
        cp->Wout = (int)M;
        rc = make_act_map(h, &cp->tmA, in.ptr, in.C, M, 1, 1, h->planes, in.plane(), 128, 1, 1);
        if (!rc && in2) rc = make_act_map(h, &cp->tmA2, in2->ptr, in2->C, M, 1, 1, h->planes, in2->plane(), 128, 1, 1);
    } else {
        // pick the patch shape with the fewest wasted rows
        double best = -1;
        tw = 16;
        const int smax = in2 ? (L.stride2 > L.stride ? L.stride2 : L.stride) : L.stride;
        for (int c = 128; c >= 1; c >>= 1) {
            const int t_h = 128 / c;
            if (c * smax > 256 || t_h * smax > 256) continue;
            if (up && (c / 2 + 2) * (t_h / 2 + 2) > 128) continue;  // the low-resolution patch must fit one ring slot
            const double util = ((double)Wo * Ho) / ((double)((Wo + c - 1) / c) * c * ((Ho + t_h - 1) / t_h) * t_h);
            if (util > best + 1e-9) {
                best = util;
                tw = c;
            }
        }
        th = 128 / tw;
        tiles_x = (Wo + tw - 1) / tw;
        tiles_y = (Ho + th - 1) / th;
        nimg = N;
        cp->Hout = Ho;
        cp->Wout = Wo;
        rc = make_act_map(h, &cp->tmA, in.ptr, in.C, in.W, in.H, N, h->planes, in.plane(), tw * L.stride,
                          th * L.stride, L.stride);
        if (!rc && in2)
            rc = make_act_map(h, &cp->tmA2, in2->ptr, in2->C, in2->W, in2->H, N, h->planes, in2->plane(),
                              tw * L.stride2, th * L.stride2, L.stride2);
    }
    if (rc) return rc;
    int twl = 0;
    while ((1 << twl) < tw) twl++;
    cp->Nimg = nimg;
    cp->tw_log2 = twl;
    cp->th = th;
    cp->tiles_x = tiles_x;
    cp->tiles_y = tiles_y;
    const long long m_tiles = (long long)tiles_x * tiles_y * nimg;
    // Tile shape from a coarse model, the starting point of the autotuner and the choice when it is off: a tile's main
    // loop costs about num_kb x (relative wgmma time of a 128 x c tile) and every tile pays an epilogue.  The two consumer
    // warpgroups overlap one tile's epilogue with the next tile's main loop, but a CTA's last epilogue and the epilogues
    // of short-K tiles (epilogue longer than a main loop) stay exposed, so the model keeps time ~ waves x (main loop +
    // epilogue).  Near-ties go to the wider tile.  The model only decides geometries that neither the committed tile table
    // (smap_b200/tiles/h100.tsv, measured with this kernel by tools/make_tile_table.py) nor the autotuner covers.
    int bn = 0, cg = 1;
    {
        const int num_kb = L.k * L.k * (L.Cin / 64) + L.Cin2 / 64;
        double best = 1e30;
        const int cands[3] = {128, 64, 32};
        for (int c : cands) {
            if (L.Cout_pad % c) continue;
            const double kb_cost = c == 128 ? 1.0 : c == 64 ? 0.6 : 0.4;
            const int n_extra = (res || up ? 1 : 0) + (post1 ? 1 : 0) + (post2 ? 1 : 0);
            const double epi = (c / 32) * (0.5 + 0.2 * n_extra + (up ? 0.5 : 0.0));
            const long long units = m_tiles * (L.Cout_pad / c);
            const double waves = (double)((units + h->sm_count - 1) / h->sm_count);
            double t = waves * (num_kb * kb_cost + epi);
            t *= (c == 64 ? 1.05 : c == 32 ? 1.10 : 1.0);
            if (t < best - 1e-9) best = t, bn = c;
        }
        if (!bn) return fail(h, -30, "conv " + L.name + ": no tile shape for Cout_pad " + std::to_string(L.Cout_pad));
    }
    if (force_bn) {  // autotuner / tile table override
        bn = force_bn;
        cg = force_cg ? force_cg : 1;
        if (L.Cout_pad % bn || !tile_shape_ok(bn, cg)) return fail(h, -31, "invalid forced tile");
    }
    if (cg_out) *cg_out = cg;
    cp->Cout = L.Cout_pad;
    cp->kh = L.stem_s2d ? 4 : L.k;
    cp->kw = L.stem_s2d ? 1 : L.k;
    cp->stride = L.stride;
    cp->pad_y = L.stem_s2d ? 2 : L.pad;
    cp->pad_x = L.stem_s2d ? 0 : L.pad;
    cp->kchunks = L.Cin / 64;
    cp->kchunks2 = L.Cin2 / 64;
    cp->stride2 = L.stride2;
    cp->n_tiles = L.Cout_pad / bn;
    cp->total_tiles = (int)(m_tiles * cp->n_tiles);
    cp->bias = L.bias_dev;
    cp->has_res = (res || up) ? 1 : 0;
    cp->n_post = (post1 ? 1 : 0) + (post2 ? 1 : 0);
    if (up) {  // fused bilinear x2 residual: the ring carries the low-resolution patch under each output tile
        cp->up_mode = 1;
        cp->up_Hi = up->H;
        cp->up_Wi = up->W;
        cp->up_pw = tw / 2 + 2;
        cp->up_ph = th / 2 + 2;
        if (up->H * 2 != Ho || up->W * 2 != Wo || up->C != L.Cout_pad || cp->up_pw * cp->up_ph > 128)
            return fail(h, -30, "conv " + L.name + ": unsupported up-residual geometry");
        rc = make_act_map(h, &cp->tmR[0], up->ptr, up->C, up->W, up->H, N, h->planes, up->plane(), cp->up_pw,
                          cp->up_ph, 1, 32);
        if (rc) return rc;
    }
    if (post2 && !post1) return fail(h, -30, "conv " + L.name + ": post2 without post1");
    cp->out = out ? out->ptr : nullptr;
    cp->out_f32 = outf ? outf->ptr : nullptr;
    cp->plane_stride = (long long)N * Ho * Wo * L.Cout_pad;
    cp->relu = relu;
    cp->sat = h->sat_dev;
    rc = make_w_map(h, &cp->tmB, L.w_dev, L.Cin + L.Cin2, L.Cout_pad, L.k * L.k, h->planes, bn);
    if (rc) return rc;
    // epilogue tiles: 32 channels x (tw x th) pixels of the output / residual planes
    int n_in = up ? 1 : 0;
    for (int which = 0; which < 4; which++) {
        const Act* t = which == 0 ? out : which == 1 ? res : which == 2 ? post1 : post2;
        if (!t) continue;
        CUtensorMap* m = which == 0 ? &cp->tmO : &cp->tmR[n_in++];
        if (flat)
            rc = make_act_map(h, m, t->ptr, L.Cout_pad, (long long)N * Ho * Wo, 1, 1, h->planes, t->plane(), 128, 1, 1, 32);
        else
            rc = make_act_map(h, m, t->ptr, L.Cout_pad, Wo, Ho, N, h->planes, t->plane(), tw, th, 1, 32);
        if (rc) return rc;
    }
    *block_n_out = bn;
    if (flops_out) *flops_out = 2.0 * N * Ho * Wo * (double)L.Cout * (L.Cin * L.k * L.k + L.Cin2);
    return 0;
}

// Tensor-core stem (7x7 s2 p3, 3 -> 64) as a 4x4 stride-1 convolution over the space-to-depth input: the A operand
// of ky-block `ay` is, for every output pixel, the 128-byte window of 4 s2d pixels x 16 channels starting at padded
// pixel ox - a *sliding* view whose dim-1 stride (32 B) is smaller than the dim-0 extent (128 B).
int setup_stem_conv(smapb_handle* h, const __nv_bfloat16* s2d, long long s2d_plane, int N, int H2, int W2, const Act& out,
                    ConvParams* cp, int* block_n_out, double* flops_out) {
    const ConvLayer& L = h->stem_tc;
    memset(cp, 0, sizeof(*cp));
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return fail(h, -20, "cuTensorMapEncodeTiled entry point not available");
    double best = -1;
    int tw = 16;
    for (int c = 128; c >= 1; c >>= 1) {
        const int t_h = 128 / c;
        const double util = ((double)W2 * H2) / ((double)((W2 + c - 1) / c) * c * ((H2 + t_h - 1) / t_h) * t_h);
        if (util > best + 1e-9) best = util, tw = c;
    }
    const int th = 128 / tw;
    const long long WP = W2 + 3;
    cuuint64_t dims[5] = {64, (cuuint64_t)W2, (cuuint64_t)H2, (cuuint64_t)N, (cuuint64_t)h->planes};
    cuuint64_t strides[4] = {32, (cuuint64_t)WP * 32, (cuuint64_t)H2 * WP * 32, (cuuint64_t)s2d_plane * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)tw, (cuuint32_t)th, 1, 1};
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(&cp->tmA, elem_dtype(h), 5, (void*)s2d, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(h, -22, "sliding-window tensor map rejected: " + std::to_string((int)r));
    int twl = 0;
    while ((1 << twl) < tw) twl++;
    cp->Hout = H2, cp->Wout = W2, cp->Nimg = N;
    cp->tw_log2 = twl, cp->th = th;
    cp->tiles_x = (W2 + tw - 1) / tw, cp->tiles_y = (H2 + th - 1) / th;
    cp->Cout = 64;
    cp->kh = 4, cp->kw = 1, cp->stride = 1, cp->pad_y = 2, cp->pad_x = 0;
    cp->kchunks = 1;
    cp->n_tiles = 1;
    cp->total_tiles = cp->tiles_x * cp->tiles_y * N;
    cp->bias = L.bias_dev;
    cp->out = out.ptr;
    cp->plane_stride = out.plane();
    cp->relu = 1;
    cp->sat = h->sat_dev;
    int rc = make_w_map(h, &cp->tmB, L.w_dev, 64, 64, 4, h->planes, 64);
    if (rc) return rc;
    rc = make_act_map(h, &cp->tmO, out.ptr, 64, W2, H2, N, h->planes, out.plane(), tw, th, 1, 32);
    if (rc) return rc;
    *block_n_out = 64;
    *flops_out = 2.0 * N * H2 * W2 * 64.0 * 147.0;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// weights: fold BN, repack, upload
// ------------------------------------------------------------------------------------------------
int fold_unit(smapb_handle* h, const std::string& name, std::vector<float>* wf, std::vector<float>* bf, int* Cout,
              int* Cin, int* k) {
    auto need = [&](const char* suffix) -> const std::vector<float>* {
        auto it = h->raw.find(name + suffix);
        return it == h->raw.end() ? nullptr : &it->second;
    };
    const auto* w = need(".conv.weight");
    const auto* b = need(".conv.bias");
    const auto* g = need(".bn.weight");
    const auto* beta = need(".bn.bias");
    const auto* mu = need(".bn.running_mean");
    const auto* var = need(".bn.running_var");
    if (!w || !b || !g || !beta || !mu || !var) return fail(h, -40, "missing weights for unit " + name);
    const auto& shp = h->raw_shape[name + ".conv.weight"];
    if (shp.size() != 4) return fail(h, -40, "bad weight rank for " + name);
    *Cout = (int)shp[0];
    *Cin = (int)shp[1];
    *k = (int)shp[2];
    const size_t per = (size_t)(*Cin) * (*k) * (*k);
    wf->resize(w->size());
    bf->resize(*Cout);
    for (int co = 0; co < *Cout; co++) {
        // BN eval (model/smap.py:23): y = (x - mean) / sqrt(var + 1e-5) * gamma + beta
        const double s = (double)(*g)[co] / sqrt((double)(*var)[co] + 1e-5);
        for (size_t i = 0; i < per; i++) (*wf)[co * per + i] = (float)((double)(*w)[co * per + i] * s);
        (*bf)[co] = (float)(((double)(*b)[co] - (double)(*mu)[co]) * s + (double)(*beta)[co]);
    }
    return 0;
}

// fp16 weights: a folded weight beyond the fp16 range cannot be represented (the unit needs bf16x3 or bf16)
int check_f16_range(smapb_handle* h, const std::string& unit, const float* w, size_t n) {
    for (size_t i = 0; i < n; i++)
        if (!(fabsf(w[i]) <= 65504.f)) {
            char buf[96];
            snprintf(buf, sizeof buf, "%g", (double)w[i]);
            return fail(h, -42, "fp16 precision: folded weight " + std::string(buf) + " of unit " + unit +
                                    " exceeds the fp16 range (65504); use bf16x3 or bf16");
        }
    return 0;
}

int upload_conv_layer(smapb_handle* h, ConvLayer& L, const std::vector<float>& wf, const std::vector<float>& bf) {
    const int taps = L.k * L.k;
    const int cin = L.Cin + L.Cin2;  // wf holds [Cout][Cin + Cin2][taps] (taps == 1 for fused pairs)
    const size_t plane = (size_t)taps * L.Cout_pad * cin;
    if (h->f16 && check_f16_range(h, L.name, wf.data(), wf.size())) return -42;
    std::vector<uint16_t> host(plane * h->planes, 0);
    for (int co = 0; co < L.Cout; co++)
        for (int ci = 0; ci < cin; ci++)
            for (int t = 0; t < taps; t++) {
                const float v = wf[((size_t)co * cin + ci) * taps + t];
                const uint16_t hi = h->f16 ? f32_to_f16_rn(v) : f32_to_bf16_rn(v);
                const size_t o = ((size_t)t * L.Cout_pad + co) * cin + ci;
                host[o] = hi;
                if (h->planes == 2) host[plane + o] = f32_to_bf16_rn(v - bf16_to_f32(hi));
            }
    std::vector<float> bias(L.Cout_pad, 0.f);
    for (int co = 0; co < L.Cout; co++) bias[co] = bf[co];
    if (!L.w_dev) {
        if (dev_alloc(h, &L.w_dev, host.size())) return -10;
        if (dev_alloc(h, &L.bias_dev, bias.size())) return -10;
    }
    CK(cudaMemcpy(L.w_dev, host.data(), host.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(L.bias_dev, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
    return 0;
}

int pad32(int c) { return (c + 31) / 32 * 32; }

void free_plan(Plan* plan) {
    if (plan->graph) cudaGraphExecDestroy(plan->graph);
    for (void* p : plan->allocs) cudaFree(p);
    for (Op& op : plan->ops)
        if (op.ev) cudaEventDestroy(op.ev);
    plan->allocs.clear();
    plan->ops.clear();
}

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct PlanBuilder {
    smapb_handle* h;
    Plan* plan;
    int B;
    int rc = 0;
    int cur_stream = 0;  // stream of the ops being added (0 main chain, 1 side branches)

    // record op (just pushed) as the producer of `out_ptr` and wire cross-stream waits for its inputs
    void wire(const void* out_ptr, std::initializer_list<const void*> inputs) {
        const int idx = (int)plan->ops.size() - 1;
        Op& op = plan->ops[idx];
        op.stream = cur_stream;
        op.inputs.assign(inputs.begin(), inputs.end());
        for (const void* in : inputs) {
            if (!in) continue;
            auto it = plan->producer.find(in);
            if (it == plan->producer.end()) continue;
            Op& prod = plan->ops[it->second];
            if (prod.stream != op.stream) {
                prod.record = true;
                op.waits.push_back(it->second);
            }
        }
        if (out_ptr) plan->producer[out_ptr] = idx;
        if (cur_stream == 1) plan->last_side = idx;
    }

    Act new_act(int N, int H, int W, int C) {
        Act a;
        a.N = N, a.H = H, a.W = W, a.C = C;
        void* p = nullptr;
        if (cudaMalloc(&p, (size_t)a.plane() * 2 * h->planes) != cudaSuccess) {
            rc = fail(h, -10, "cudaMalloc failed for activation tensor");
            return a;
        }
        plan->allocs.push_back(p);
        // one-time zero fill: every element is overwritten by its producer before it is read, but the producers store
        // through TMA (cp.async.bulk.tensor), which compute-sanitizer's initcheck does not track
        cudaMemset(p, 0, (size_t)a.plane() * 2 * h->planes);
        a.ptr = (__nv_bfloat16*)p;
        return a;
    }
    ActF32 new_f32(int N, int H, int W, int C) {
        ActF32 a;
        a.N = N, a.H = H, a.W = W, a.C = C;
        void* p = nullptr;
        if (cudaMalloc(&p, (size_t)N * H * W * C * 4) != cudaSuccess) {
            rc = fail(h, -10, "cudaMalloc failed for fp32 tensor");
            return a;
        }
        plan->allocs.push_back(p);
        a.ptr = (float*)p;
        return a;
    }
    // SMAPB_SERPENTINE: a conv walks its tile list in the opposite direction of the op that produced its input, so that it
    // starts with the rows written last (still in L2) instead of the ones written first (evicted by then)
    int reverse_for(const void* in_ptr) {
        if (!h->serpentine) return 0;
        auto it = plan->producer.find(in_ptr);
        if (it == plan->producer.end()) return 1;
        const Op& prod = plan->ops[it->second];
        return prod.kind == OP_CONV ? !prod.cp.reverse : 1;
    }
    const ConvLayer* layer(const std::string& name) {
        auto it = h->layers.find(name);
        if (it == h->layers.end()) {
            rc = fail(h, -41, "layer not found: " + name);
            return nullptr;
        }
        return &it->second;
    }
    // Empirical tile selection: time every valid (BLOCK_N, CG) for this layer geometry once (activation contents do not
    // matter for the timing) and keep the fastest; the cost model only provides the starting point.
    int tune(const ConvLayer& L, const Act& in, const Act* res, const Act* p1, const Act* p2, const Act* out, int relu,
             const Act* in2, const Act* up, Op* op) {
        char key[256];
        // fp16 rows carry the element type: they never match (or overwrite) a bf16 row of the same geometry
        snprintf(key, sizeof key, "%d/%d/%d k%d s%d %dx%dx%d r%d p%d u%d c2_%d s2_%d t%d%s", L.Cin, L.Cout_pad, L.Cin2, L.k,
                 L.stride, in.N, in.H, in.W, res ? 1 : 0, (p1 ? 1 : 0) + (p2 ? 1 : 0), up ? 1 : 0, L.Cin2, L.stride2,
                 h->nterms, h->f16 ? " f16" : "");
        int best_bn = 0, best_cg = 1;
        bool known = false;
        {
            std::lock_guard<std::mutex> lk(g_tiles_mu);
            auto it = g_tiles.find(key);
            // an entry this kernel has no variant for (a table written for another GPU) is measured again
            if (it != g_tiles.end() && tile_shape_ok(it->second.first, it->second.second))
                best_bn = it->second.first, best_cg = it->second.second, known = true;
        }
        if (!known && !h->autotune) return 0;  // cost model (deterministic)
        if (!known) {
            cudaEvent_t e0, e1;
            cudaEventCreate(&e0);
            cudaEventCreate(&e1);
            float best_ms = 1e30f;
            const int cand[3][2] = {{128, 1}, {64, 1}, {32, 1}};
            for (auto& c : cand) {
                if (L.Cout_pad % c[0]) continue;
                if (c[0] == 32 && L.Cout_pad > 64) continue;
                Op trial;
                int rc2 = setup_conv(h, L, in, res, p1, p2, out, nullptr, relu, &trial.cp, &trial.block_n, &trial.flops, in2,
                                     up, &trial.cg, c[0], c[1]);
                if (rc2) continue;
                float ms_best_c = 1e30f;
                for (int rep = 0; rep < 4; rep++) {
                    cudaEventRecord(e0, nullptr);
                    if (launch_conv(trial.cp, trial.block_n, h->nterms, h->f16, h->sm_count, nullptr, false) != cudaSuccess) {
                        ms_best_c = 1e30f;
                        break;
                    }
                    cudaEventRecord(e1, nullptr);
                    if (cudaEventSynchronize(e1) != cudaSuccess) return fail(h, -10, "autotune launch failed");
                    float ms = 0;
                    cudaEventElapsedTime(&ms, e0, e1);
                    if (rep > 0 && ms < ms_best_c) ms_best_c = ms;
                }
                if (ms_best_c < best_ms) best_ms = ms_best_c, best_bn = c[0], best_cg = c[1];
            }
            cudaEventDestroy(e0);
            cudaEventDestroy(e1);
            h->err.clear();
            if (!best_bn) return 0;  // keep the model's choice
            std::lock_guard<std::mutex> lk(g_tiles_mu);
            auto it = g_tiles.find(key);
            if (it == g_tiles.end() || !tile_shape_ok(it->second.first, it->second.second))
                g_tiles[key] = std::make_pair(best_bn, best_cg);  // new, or replaces an entry this kernel cannot run
            else
                best_bn = it->second.first, best_cg = it->second.second;  // another handle may have been first
        }
        if (best_bn == op->block_n && best_cg == op->cg) return 0;
        return setup_conv(h, L, in, res, p1, p2, out, nullptr, relu, &op->cp, &op->block_n, &op->flops, in2, up, &op->cg,
                          best_bn, best_cg);
    }
    Act conv(const std::string& name, const Act& in, int relu, const Act* res = nullptr, const Act* p1 = nullptr,
             const Act* p2 = nullptr, const Act* in2 = nullptr, const Act* up = nullptr) {
        Act out;
        if (rc) return out;
        const ConvLayer* L = layer(name);
        if (!L) return out;
        const int Ho = (in.H + 2 * L->pad - L->k) / L->stride + 1, Wo = (in.W + 2 * L->pad - L->k) / L->stride + 1;
        out = new_act(in.N, Ho, Wo, L->Cout_pad);
        if (rc) return out;
        Op op;
        op.kind = OP_CONV;
        rc = setup_conv(h, *L, in, res, p1, p2, &out, nullptr, relu, &op.cp, &op.block_n, &op.flops, in2, up, &op.cg);
        if (!rc) rc = tune(*L, in, res, p1, p2, &out, relu, in2, up, &op);
        op.name = name;
        op.cp.reverse = reverse_for(in.ptr);
        op.dims[0] = out.N, op.dims[1] = out.H, op.dims[2] = out.W, op.dims[3] = out.C;
        plan->ops.push_back(op);
        wire(out.ptr, {in.ptr, res ? res->ptr : nullptr, p1 ? p1->ptr : nullptr, p2 ? p2->ptr : nullptr,
                       in2 ? in2->ptr : nullptr, up ? up->ptr : nullptr});
        plan->n_conv++;
        plan->conv_flops += op.flops;
        return out;
    }
    ActF32 conv_f32(const std::string& name, const Act& in) {
        ActF32 out;
        if (rc) return out;
        const ConvLayer* L = layer(name);
        if (!L) return out;
        out = new_f32(in.N, in.H, in.W, L->Cout_pad);
        if (rc) return out;
        Op op;
        op.kind = OP_CONV;
        rc = setup_conv(h, *L, in, nullptr, nullptr, nullptr, nullptr, &out, 0, &op.cp, &op.block_n, &op.flops);
        op.name = name;
        op.cp.reverse = reverse_for(in.ptr);
        op.dims[0] = out.N, op.dims[1] = out.H, op.dims[2] = out.W, op.dims[3] = out.C;
        plan->ops.push_back(op);
        wire(out.ptr, {in.ptr});
        plan->n_conv++;
        plan->conv_flops += op.flops;
        return out;
    }
};

int build_plan(smapb_handle* h, int B, Plan** out_plan, int instance = 0) {
    const int key = B + 100000 * instance;  // instance > 0: an independent copy (own activations) for a second stream
    auto it = h->plans.find(key);
    if (it != h->plans.end()) {
        *out_plan = it->second.get();
        return 0;
    }
    std::unique_ptr<Plan> plan(new Plan());
    plan->B = B;
    PlanBuilder pb{h, plan.get(), B};
    const int H = h->in_h, W = h->in_w;
    static const int LAYERS[4] = {3, 4, 6, 3};
    // stem + maxpool (model/smap.py:88-92)
    Act stem = pb.new_act(B, H / 2, W / 2, 64);
    {
        // tensor-core stem over the space-to-depth input when the driver accepts the sliding-window TMA view,
        // otherwise the fp32 CUDA-core stem kernel (both are GPU paths; SMAPB_STEM=cuda forces the latter)
        bool tc = h->stem_tc_ok != 0 && !(getenv("SMAPB_STEM") && !strcmp(getenv("SMAPB_STEM"), "cuda"));
        if (tc) {
            Act s2d;  // storage [plane][B][H/2][W/2+3][16]
            s2d.N = B, s2d.H = H / 2, s2d.W = W / 2 + 3, s2d.C = 16;
            void* p = nullptr;
            if (cudaMalloc(&p, (size_t)s2d.plane() * 2 * h->planes) != cudaSuccess)
                return fail(h, -10, "cudaMalloc failed for the s2d input");
            plan->allocs.push_back(p);
            cudaMemset(p, 0, (size_t)s2d.plane() * 2 * h->planes);
            s2d.ptr = (__nv_bfloat16*)p;
            Op oc;
            oc.kind = OP_CONV;
            int rc2 = setup_stem_conv(h, s2d.ptr, s2d.plane(), B, H / 2, W / 2, stem, &oc.cp, &oc.block_n, &oc.flops);
            if (rc2 == -22) {
                h->stem_tc_ok = 0;
                tc = false;
            } else if (rc2) {
                return rc2;
            } else {
                h->stem_tc_ok = 1;
                Op os;
                os.kind = OP_S2D;
                os.name = "top.s2d";
                oc.name = "top.conv";
                os.out = s2d;
                oc.dims[0] = stem.N, oc.dims[1] = stem.H, oc.dims[2] = stem.W, oc.dims[3] = stem.C;
                plan->ops.push_back(os);
                pb.wire(s2d.ptr, {});
                plan->ops.push_back(oc);
                pb.wire(stem.ptr, {s2d.ptr});
                plan->n_conv++;
                plan->conv_flops += oc.flops;
            }
        }
        if (!tc) {
            Op op;
            op.kind = OP_STEM;
            op.name = "top.conv";
            op.out = stem;
            plan->ops.push_back(op);
            pb.wire(stem.ptr, {});
        }
    }
    Act x = pb.new_act(B, H / 4, W / 4, 64);
    {
        Op op;
        op.kind = OP_MAXPOOL;
        op.name = "top.maxpool";
        op.a = stem;
        op.out = x;
        plan->ops.push_back(op);
        pb.wire(x.ptr, {stem.ptr});
    }
    Act skip1[4], skip2[4];
    ActF32 res[4], resd3, resrd3;
    std::string name_d, name_rd;
    for (int s = 0; s < 3 && !pb.rc; s++) {
        const std::string pre = "stage" + std::to_string(s) + ".";
        const bool gen_skip = s != 2;
        Act feats[4];
        Act t = x;
        for (int li = 0; li < 4; li++) {
            for (int b = 0; b < LAYERS[li]; b++) {
                const std::string p = pre + "downsample.layer" + std::to_string(li + 1) + "." + std::to_string(b) + ".";
                Act o1 = pb.conv(p + "conv_bn_relu1", t, 1);
                Act o2 = pb.conv(p + "conv_bn_relu2", o1, 1);
                const bool last = (b == LAYERS[li] - 1) && s > 0;
                if (b == 0 && !getenv("SMAPB_NO_FUSE_DS")) {
                    // relu(conv3(o2) + downsample(x)) as one K-concatenated GEMM
                    t = pb.conv(p + "fused_conv3_downsample", o2, 1, nullptr, nullptr, nullptr, &t);
                } else if (b == 0) {  // debug: separate downsample + residual
                    Act idn = pb.conv(p + "downsample", t, 0);
                    t = pb.conv(p + "conv_bn_relu3", o2, 1, &idn);
                } else {
                    // out = relu(conv3 + x) [ + skip1 + skip2 ]   (model/smap.py:74-75,143)
                    t = pb.conv(p + "conv_bn_relu3", o2, 1, &t, last ? &skip1[li] : nullptr,
                                last ? &skip2[li] : nullptr);
                }
            }
            feats[li] = t;
        }
        Act up_x;
        Act sk1[4], sk2[4];
        Act cross;
        for (int ind = 0; ind < 4 && !pb.rc; ind++) {
            const std::string p = pre + "upsample.up" + std::to_string(ind + 1) + ".";
            const Act& xin = feats[3 - ind];
            Act out;
            if (ind == 0) {
                out = pb.conv(p + "u_skip", xin, 1);
            } else {
                // out = relu(u_skip(x) + bilinear_x2(up_conv(up_x))): the 1x1 up_conv is commuted in front of the
                // interpolation (both linear, bilinear weights sum to 1) and the interpolation + add + ReLU run in the
                // u_skip epilogue
                Act tl = pb.conv(p + "up_conv", up_x, 0);
                if (!getenv("SMAPB_NO_FUSE_UP")) {
                    out = pb.conv(p + "u_skip", xin, 1, nullptr, nullptr, nullptr, nullptr, &tl);
                } else {  // debug: separate bilinear + add + relu kernel
                    Act a = pb.conv(p + "u_skip", xin, 0);
                    out = pb.new_act(a.N, a.H, a.W, a.C);
                    Op op;
                    op.kind = OP_UPADD;
                    op.a = a;
                    op.b = tl;
                    op.out = out;
                    plan->ops.push_back(op);
                    pb.wire(out.ptr, {a.ptr, tl.ptr});
                }
            }
            // Side branches (heads, skip convs) hang off `out` / `xin` and are only needed much later: they go to the
            // second stream and overlap the main chain, filling SMs that small layers leave idle.
            pb.cur_stream = h->two_streams ? 1 : 0;
            // heads: only those that reach the returned tensors (model/smap.py:418-419) are computed
            if (s == 2 && ind >= 1) {
                Act r1 = pb.conv(p + "res_conv1", out, 1);
                res[ind] = pb.conv_f32(p + "res_conv2", r1);
            }
            if (s == 2 && ind == 3) {
                Act d1 = pb.conv(p + "res_d_conv1", out, 1);
                resd3 = pb.conv_f32(p + "res_d_conv2.tapexp", d1);
                Act rd1 = pb.conv(p + "res_rd_conv1", out, 1);
                resrd3 = pb.conv_f32(p + "res_rd_conv2.tapexp", rd1);
                name_d = p + "res_d_conv2";
                name_rd = p + "res_rd_conv2";
            }
            if (gen_skip) {
                sk1[ind] = pb.conv(p + "skip1", xin, 1);
                sk2[ind] = pb.conv(p + "skip2", out, 1);
                pb.cur_stream = 0;
                if (ind == 3) cross = pb.conv(p + "cross_conv", out, 1);
            }
            pb.cur_stream = 0;
            up_x = out;
        }
        for (int li = 0; li < 4; li++) {  // skip lists are finest-first (model/smap.py:281-282)
            skip1[li] = sk1[3 - li];
            skip2[li] = sk2[3 - li];
        }
        x = cross;
    }
    if (pb.rc) {
        free_plan(plan.get());
        return pb.rc;
    }
    {
        Op op;
        op.kind = OP_HEADMERGE;
        op.name = "head_merge(res4+res3+res2)";
        op.f4 = res[3], op.f3 = res[2], op.f2 = res[1];
        op.cout = 43;
        op.which_out = 0;
        plan->ops.push_back(op);
        pb.wire(nullptr, {res[3].ptr, res[2].ptr, res[1].ptr});
        Op od;
        od.kind = OP_TAPSUM;
        od.name = "tapsum(res_d)";
        od.f4 = resd3;
        od.cout = 14;
        od.which_out = 1;
        od.bias = h->layers[name_d].bias_dev;
        plan->ops.push_back(od);
        pb.wire(nullptr, {resd3.ptr});
        Op ord_;
        ord_.kind = OP_TAPSUM;
        ord_.name = "tapsum(res_rd)";
        ord_.f4 = resrd3;
        ord_.cout = 1;
        ord_.which_out = 2;
        ord_.bias = h->layers[name_rd].bias_dev;
        plan->ops.push_back(ord_);
        pb.wire(nullptr, {resrd3.ptr});
        // the main stream must not run ahead of the side stream into the next forward: the last op joins it
        if (plan->last_side >= 0) {
            plan->ops[plan->last_side].record = true;
            plan->ops.back().waits.push_back(plan->last_side);
        }
    }
    for (Op& op : plan->ops)
        if (op.record) cudaEventCreateWithFlags(&op.ev, cudaEventDisableTiming);
    *out_plan = plan.get();
    h->plans[key] = std::move(plan);
    return 0;
}

int run_plan(smapb_handle* h, Plan* plan, const float* imgs, float* hm2d, float* detd, float* rootd,
             cudaStream_t st) {
    const int B = plan->B;
    const int T = h->planes;
    prof_mark(h, PK_START, st);
    // profiling serialises everything on one stream (per-op event deltas); otherwise side-branch ops run on the
    // handle's second stream, ordered against the main chain by events on exactly the tensors they exchange
    const bool multi = !h->profiling && h->aux_stream != nullptr;
    cudaStream_t const main_st = st;
    static const int stop_after = getenv("SMAPB_DEBUG_STOP") ? atoi(getenv("SMAPB_DEBUG_STOP")) : 1 << 30;
    int op_idx = 0;
    for (const Op& op : plan->ops) {
        if (op_idx++ >= stop_after) break;
        st = (multi && op.stream == 1) ? h->aux_stream : main_st;
        if (multi)
            for (int w : op.waits) CK(cudaStreamWaitEvent(st, plan->ops[w].ev, 0));
        if (h->nvtx_ops) nvtxRangePushA(op.name.empty() ? "smapb.op" : op.name.c_str());
        switch (op.kind) {
            case OP_STEM:
                CK(launch_stem(imgs, h->stem_w, h->stem_b, B, h->in_h, h->in_w, op.out.ptr, op.out.plane(), T, st, h->f16,
                               h->sat_dev));
                prof_mark(h, PK_STEM, st, "stem7x7");
                break;
            case OP_S2D:
                CK(launch_s2d(imgs, B, h->in_h, h->in_w, op.out.ptr, op.out.plane(), T, st, h->f16, h->sat_dev));
                prof_mark(h, PK_STEM, st, "s2d");
                break;
            case OP_MAXPOOL:
                CK(launch_maxpool(op.a.ptr, op.a.plane(), B, op.a.H, op.a.W, op.a.C, op.out.ptr, op.out.plane(), T, st,
                                  h->f16));
                prof_mark(h, PK_STEM, st, "maxpool");
                break;
            case OP_CONV:
                if (h->profiling && h->roles_dev && h->roles_used < ROLES_CAP) {
                    ConvParams cp = op.cp;  // same launch with the wait-cycle counters of every warp role switched on
                    cp.dbg = h->roles_dev + 16 * h->roles_used++;
                    CK(launch_conv(cp, op.block_n, h->nterms, h->f16, h->sm_count - h->sm_reserve, st, h->use_pdl));
                } else {
                    CK(launch_conv(op.cp, op.block_n, h->nterms, h->f16, h->sm_count - h->sm_reserve, st, h->use_pdl));
                }
                if (h->profiling) {
                    char d[160];
                    snprintf(d, sizeof d, "conv k%dx%d s%d cin%d cout%d out%dx%d bn%d cg%d tiles%d", op.cp.kh, op.cp.kw,
                             op.cp.stride, op.cp.kchunks * 64, op.cp.Cout, op.cp.Hout, op.cp.Wout, op.block_n, op.cg,
                             op.cp.total_tiles);
                    prof_mark(h, PK_CONV, st, d, op.flops);
                    if (h->roles_dev) h->roles_desc.push_back(op.name + "," + d);
                }
                break;
            case OP_UPADD:
                CK(launch_upadd_relu(op.a.ptr, op.a.plane(), op.b.ptr, op.b.plane(), B, op.a.H, op.a.W, op.b.H, op.b.W,
                                     op.a.C, op.out.ptr, op.out.plane(), T, st, h->f16, h->sat_dev));
                prof_mark(h, PK_ELEM, st, "upadd_relu");
                break;
            case OP_TAPSUM: {
                float* dst = op.which_out == 1 ? detd : rootd;
                CK(launch_tapsum(op.f4.ptr, op.bias, B, op.f4.H, op.f4.W, op.f4.C, op.cout, dst, st));
                prof_mark(h, PK_ELEM, st, "tapsum");
                break;
            }
            case OP_HEADMERGE: {
                float* dst = op.which_out == 0 ? hm2d : op.which_out == 1 ? detd : rootd;
                CK(launch_head_merge(op.f4.ptr, op.f3.ptr, op.f2.ptr, B, op.f4.H, op.f4.W, op.f3.H, op.f3.W, op.f2.H,
                                     op.f2.W, op.f4.C, op.cout, dst, st));
                prof_mark(h, PK_ELEM, st, "head_merge");
                break;
            }
        }
        if (h->nvtx_ops) nvtxRangePop();
        h->launches++;
        if (multi && op.record) CK(cudaEventRecord(op.ev, st));
        static const bool debug_sync = getenv("SMAPB_DEBUG_SYNC") != nullptr;
        if (debug_sync) CK(cudaStreamSynchronize(st));
    }
    return 0;
}

// debug: the output tensor of an op that smapb_debug_dump / smapb_debug_checksums report (null: the op has no dumped
// output) and its size in bytes (both bf16 planes, or fp32).  Both entry points number the dumped ops with this predicate.
const void* dumped_output(const smapb_handle* h, const Op& op, long long* bytes) {
    if (op.kind == OP_CONV && op.cp.out) return *bytes = op.cp.plane_stride * h->planes * 2, op.cp.out;
    if (op.kind == OP_CONV && op.cp.out_f32) return *bytes = op.cp.plane_stride * 4, op.cp.out_f32;
    if (op.out.ptr) return *bytes = op.out.plane() * h->planes * 2, op.out.ptr;
    *bytes = 0;
    return nullptr;
}

// debug: one self-describing line per dumped op (format: include/smap_b200_debug.h).  `dump_idx` maps every dumped
// output tensor to its dump index, so that the op's inputs can be named by index.
std::string debug_op_desc(const smapb_handle* h, const Op& op, const std::map<const void*, int>& dump_idx) {
    static const char* const CONV_ROLES[6] = {"in", "res", "p1", "p2", "in2", "up"};
    const bool is_conv = op.kind == OP_CONV;
    const bool stem_tc = is_conv && op.cp.kh == 4 && op.cp.kw == 1;
    const char* kind = is_conv ? (stem_tc ? "stem_tc" : op.cp.out ? "conv" : "conv_f32")
                       : op.kind == OP_STEM ? "stem" : op.kind == OP_S2D ? "s2d" : op.kind == OP_MAXPOOL ? "maxpool"
                       : op.kind == OP_UPADD ? "upadd" : "other";
    std::string s = "name=" + (op.name.empty() ? std::string("?") : op.name) + " kind=" + kind;
    if (op.kind == OP_STEM || op.kind == OP_S2D) s += " in=x";  // the network input image
    for (size_t r = 0; r < op.inputs.size(); r++) {
        if (!op.inputs[r]) continue;
        const char* role = is_conv ? (r < 6 ? CONV_ROLES[r] : "?") : (r == 0 ? "a" : "b");
        auto it = dump_idx.find(op.inputs[r]);
        s += std::string(" ") + role + "=" + (it == dump_idx.end() ? std::string("?") : std::to_string(it->second));
    }
    char buf[320];
    if (is_conv) {
        snprintf(buf, sizeof buf,
                 " tw=%d rev=%d k=%dx%d s=%d pad=%dx%d cin=%d cin2=%d s2=%d cout=%d out=%dx%dx%dx%d bn=%d cg=%d relu=%d "
                 "hasres=%d post=%d upmode=%d tiles=%d nterms=%d",
                 1 << op.cp.tw_log2, op.cp.reverse, op.cp.kh, op.cp.kw, op.cp.stride, op.cp.pad_y, op.cp.pad_x,
                 op.cp.kchunks * 64, op.cp.kchunks2 * 64, op.cp.stride2, op.cp.Cout, op.dims[0], op.dims[1], op.dims[2],
                 op.dims[3], op.block_n, op.cg, op.cp.relu, op.cp.has_res, op.cp.n_post, op.cp.up_mode,
                 op.cp.total_tiles, h->nterms);
    } else {
        snprintf(buf, sizeof buf, " out=%dx%dx%dx%d nterms=%d", op.out.N, op.out.H, op.out.W, op.out.C, h->nterms);
    }
    return s + buf + (h->f16 ? " dtype=f16" : "");
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {
#pragma GCC visibility push(default)

int smapb_version(void) { return 200; }

const char* smapb_last_error(const smapb_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int smapb_create(smapb_handle** out, int device, int max_batch, int in_h, int in_w) {
    if (!out) return -1;
    *out = nullptr;
    if (max_batch < 1 || in_h % 32 || in_w % 32 || in_h < 32 || in_w < 32) {
        g_create_error = "smapb_create: max_batch >= 1 and in_h, in_w multiples of 32 required";
        return -1;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device >= ndev) {
        g_create_error = std::string("smapb_create: no usable CUDA device (") + cudaGetErrorString(e) + ")";
        return -2;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    if (prop.major != 9 || prop.minor != 0) {
        g_create_error = "smapb_create: this library contains sm_90a code only (device is sm_" +
                         std::to_string(prop.major) + std::to_string(prop.minor) + ")";
        return -3;
    }
    cudaSetDevice(device);
    smapb_handle* h = new smapb_handle();
    h->device = device;
    h->max_batch = max_batch;
    h->in_h = in_h, h->in_w = in_w;
    h->h = in_h / 4, h->w = in_w / 4;
    h->sm_count = prop.multiProcessorCount;
    // SMs left free by the persistent conv grids (see smapb_comm_create): a conv CTA takes a whole SM (227 KB of shared
    // memory), so any other resident CTA - a spinning NCCL channel, the other handle's grouping kernel - pushes one conv
    // CTA into a second wave
    if (getenv("SMAPB_SM_RESERVE")) h->sm_reserve = std::max(0, std::min(32, atoi(getenv("SMAPB_SM_RESERVE"))));
    const size_t hw = (size_t)h->h * h->w;
    const size_t MB = max_batch;
    int rc = 0;
    rc |= dev_alloc(h, &h->peaks, MB * NJ * (MAXP + 1) * 3);
    rc |= dev_alloc(h, &h->scores, MB * NL * MAXP * MAXP);
    rc |= dev_alloc(h, &h->bodies, MB * MAXP * NJ * 4);
    rc |= dev_alloc(h, &h->counts, MB);
    rc |= dev_alloc(h, &h->nms_masks, nms_mask_words(max_batch, h->h, h->w));
    rc |= dev_alloc(h, &h->imgs_dev, MB * 3 * in_h * in_w);
    rc |= dev_alloc(h, &h->hm, MB * NC2D * hw);
    rc |= dev_alloc(h, &h->detd, MB * NL * hw);
    rc |= dev_alloc(h, &h->rootd, MB * hw);
    rc |= dev_alloc(h, &h->scales_dev, MB * SMAPB_SCALE_LEN);
    rc |= dev_alloc(h, &h->records_dev, MB);
    rc |= dev_alloc(h, &h->sat_dev, 1);
    if (!rc && cudaMemset(h->sat_dev, 0, sizeof(unsigned long long)) != cudaSuccess) rc = -10;
    if (rc) {
        g_create_error = h->err;
        delete h;
        return -10;
    }
    if (cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->bridge_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->bridge_out, cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreateWithFlags(&h->aux_stream, cudaStreamNonBlocking) != cudaSuccess) {
        g_create_error = "smapb_create: stream / event creation failed";
        smapb_destroy(h);
        return -10;
    }
    const char* aerr = nullptr;
    // association kernels stage whole planes in shared memory; larger maps are rejected at call time
    if (assoc_configure(h->h, h->w, &aerr) != 0) h->err = aerr ? aerr : "assoc_configure failed";
    *out = h;
    return 0;
}

void smapb_destroy(smapb_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (auto& kv : h->plans) free_plan(kv.second.get());
    for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
    for (auto& S : h->slots) {
        cudaFree(S.imgs);
        cudaFree(S.scales);
        cudaFree(S.records);
        cudaFree(S.records_all);
        if (S.h2d) cudaEventDestroy(S.h2d);
        if (S.done) cudaEventDestroy(S.done);
        if (S.rec_ready) cudaEventDestroy(S.rec_ready);
    }
    if (h->comm && h->comm_owned && nccl_api().CommDestroy) nccl_api().CommDestroy(h->comm);
    if (h->gather_stream) cudaStreamDestroy(h->gather_stream);
    for (int i = 0; i < 2; i++) {
        if (h->rec_ready[i]) cudaEventDestroy(h->rec_ready[i]);
        if (h->gather_done[i]) cudaEventDestroy(h->gather_done[i]);
        cudaFree(h->rec_buf[i]);
    }
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    if (h->aux_stream) cudaStreamDestroy(h->aux_stream);
    if (h->bridge_in) cudaEventDestroy(h->bridge_in);
    if (h->bridge_out) cudaEventDestroy(h->bridge_out);
    for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
    for (auto& kv : h->layers) {
        cudaFree(kv.second.w_dev);
        cudaFree(kv.second.bias_dev);
    }
    cudaFree(h->stem_tc.w_dev);
    cudaFree(h->stem_tc.bias_dev);
    void* ptrs[] = {h->peaks, h->scores, h->bodies, h->counts, h->imgs_dev, h->imgs_flip, h->hm, h->hm_flip, h->detd,
                    h->rootd, h->scratch_detd, h->scratch_rootd, h->scales_dev, h->records_dev, h->stem_w, h->stem_b,
                    h->gather_dev, h->gt_dist, h->nms_masks, h->sat_dev};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (h->refine_buf) cudaFree(h->refine_buf);
    if (h->roles_dev) cudaFree(h->roles_dev);
    if (h->pre_stage) cudaFree(h->pre_stage);
    for (auto& e : h->pre_cache) cudaFree(e.second.buf);
    delete h;
}

int smapb_load_weight(smapb_handle* h, const char* key, const float* host, const int64_t* shape, int ndim) {
    if (!h || !key || !host) return -1;
    const std::string k(key);
    if (k.size() > 19 && k.compare(k.size() - 19, 19, "num_batches_tracked") == 0) return 0;
    size_t n = 1;
    std::vector<int64_t> shp;
    for (int i = 0; i < ndim; i++) {
        n *= (size_t)shape[i];
        shp.push_back(shape[i]);
    }
    h->raw[k].assign(host, host + n);
    h->raw_shape[k] = shp;
    h->finalized = false;
    return 0;
}

int smapb_finalize_weights(smapb_handle* h, int precision) {
    if (!h) return -1;
    if (precision != SMAPB_PREC_BF16X3 && precision != SMAPB_PREC_BF16 && precision != SMAPB_PREC_FP16)
        return fail(h, -1, "unknown precision");
    cudaSetDevice(h->device);
    // a new weight set invalidates cached plans (they hold tensor maps over the old weight buffers only if
    // buffers are re-allocated; buffers are reused in place, but the plane count may change)
    const int new_planes = precision == SMAPB_PREC_BF16X3 ? 2 : 1;
    h->finalized = false;
    for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
    h->graphs.clear();
    h->eager_runs.clear();
    if (new_planes != h->planes || !h->plans.empty()) {
        cudaDeviceSynchronize();
        for (auto& kv : h->plans) free_plan(kv.second.get());
        h->plans.clear();
        for (auto& kv : h->layers) {
            cudaFree(kv.second.w_dev);
            cudaFree(kv.second.bias_dev);
        }
        h->layers.clear();
        cudaFree(h->stem_tc.w_dev);
        cudaFree(h->stem_tc.bias_dev);
        h->stem_tc.w_dev = nullptr;
        h->stem_tc.bias_dev = nullptr;
    }
    h->nterms = precision == SMAPB_PREC_BF16X3 ? 3 : 1;
    h->planes = new_planes;
    h->f16 = precision == SMAPB_PREC_FP16;
    // unit names: every "<name>.conv.weight" key
    std::vector<std::string> units;
    for (auto& kv : h->raw) {
        const std::string& k = kv.first;
        const std::string suf = ".conv.weight";
        if (k.size() > suf.size() && k.compare(k.size() - suf.size(), suf.size(), suf) == 0)
            units.push_back(k.substr(0, k.size() - suf.size()));
    }
    if (units.empty()) return fail(h, -40, "no weights loaded");
    std::map<std::string, std::pair<std::vector<float>, std::vector<float>>> folded;  // 1x1 units of bottleneck pairs
    for (const std::string& name : units) {
        std::vector<float> wf, bf;
        int Cout, Cin, k;
        int rc = fold_unit(h, name, &wf, &bf, &Cout, &Cin, &k);
        if (rc) return rc;
        if (name.find(".downsample.layer") != std::string::npos &&
            (name.find(".0.conv_bn_relu3") != std::string::npos ||
             (name.size() > 13 && name.compare(name.size() - 13, 13, ".0.downsample") == 0)))
            folded[name] = {wf, bf};
        if (name.find("res_d_conv2") != std::string::npos || name.find("res_rd_conv2") != std::string::npos)
            folded[name] = {wf, bf};
        if (name == "top.conv") {
            if (Cin != 3 || Cout != 64 || k != 7) return fail(h, -40, "top.conv must be 3->64 7x7");
            std::vector<float> w2(147 * 64);
            for (int co = 0; co < 64; co++)
                for (int ci = 0; ci < 3; ci++)
                    for (int ky = 0; ky < 7; ky++)
                        for (int kx = 0; kx < 7; kx++)
                            w2[((ky * 7 + kx) * 3 + ci) * 64 + co] = wf[((co * 3 + ci) * 7 + ky) * 7 + kx];
            if (!h->stem_w) {
                if (dev_alloc(h, &h->stem_w, w2.size())) return -10;
                if (dev_alloc(h, &h->stem_b, 64)) return -10;
            }
            CK(cudaMemcpy(h->stem_w, w2.data(), w2.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(h->stem_b, bf.data(), 64 * 4, cudaMemcpyHostToDevice));
            {  // tensor-core stem weights: [plane][ay][co][k], k = ax*16 + (by*2+bx)*3 + c; ky = 2*ay+by-1, kx = 2*ax+bx-1
                ConvLayer& S = h->stem_tc;
                S.name = "top.conv(s2d)";
                S.Cin = 64, S.Cout = 64, S.Cout_pad = 64, S.k = 1, S.stride = 1, S.pad = 0, S.stem_s2d = true;
                const size_t plane = (size_t)4 * 64 * 64;
                if (h->f16 && check_f16_range(h, name, wf.data(), wf.size())) return -42;
                std::vector<uint16_t> host(plane * h->planes, 0);
                for (int co = 0; co < 64; co++)
                    for (int ay = 0; ay < 4; ay++)
                        for (int ax = 0; ax < 4; ax++)
                            for (int by = 0; by < 2; by++)
                                for (int bx = 0; bx < 2; bx++)
                                    for (int c = 0; c < 3; c++) {
                                        const int ky = 2 * ay + by - 1, kx = 2 * ax + bx - 1;
                                        if (ky < 0 || ky > 6 || kx < 0 || kx > 6) continue;
                                        const float v = wf[((co * 3 + c) * 7 + ky) * 7 + kx];
                                        const uint16_t hi = h->f16 ? f32_to_f16_rn(v) : f32_to_bf16_rn(v);
                                        const size_t o = ((size_t)ay * 64 + co) * 64 + ax * 16 + (by * 2 + bx) * 3 + c;
                                        host[o] = hi;
                                        if (h->planes == 2) host[plane + o] = f32_to_bf16_rn(v - bf16_to_f32(hi));
                                    }
                if (!S.w_dev) {
                    if (dev_alloc(h, &S.w_dev, host.size())) return -10;
                    if (dev_alloc(h, &S.bias_dev, 64)) return -10;
                }
                CK(cudaMemcpy(S.w_dev, host.data(), host.size() * 2, cudaMemcpyHostToDevice));
                CK(cudaMemcpy(S.bias_dev, bf.data(), 64 * 4, cudaMemcpyHostToDevice));
            }
            continue;
        }
        ConvLayer& L = h->layers[name];
        L.name = name;
        L.Cin = Cin;
        L.Cout = Cout;
        L.Cout_pad = pad32(Cout);
        L.k = k;
        L.pad = k / 2;
        // stride: first 3x3 / downsample of layer2..4 (model/smap.py:103-108,124-136)
        L.stride = 1;
        {
            const size_t pl = name.find(".downsample.layer");
            if (pl != std::string::npos) {
                const int li = name[pl + 17] - '0';
                const size_t pb = name.find('.', pl + 18);
                const int blk = atoi(name.c_str() + pl + 19);
                (void)pb;
                const bool first = blk == 0;
                const bool is_c2 = name.find("conv_bn_relu2") != std::string::npos;
                const bool is_ds = name.size() > 11 && name.compare(name.size() - 11, 11, ".downsample") == 0;
                if (li >= 2 && first && (is_c2 || is_ds)) L.stride = 2;
            }
        }
        int rc2 = upload_conv_layer(h, L, wf, bf);
        if (rc2) return rc2;
    }
    // First bottleneck of every layer: out = relu(conv3(o2) + downsample(x)) (model/smap.py:70-75) is ONE GEMM over
    // the K-concatenated inputs [o2 | x] with weights [W3 | Wds] and bias b3 + bds: the downsample tensor is never
    // written to HBM and never re-read as a residual.
    for (auto& kv : folded) {
        const std::string& n3 = kv.first;
        const size_t pos = n3.find(".0.conv_bn_relu3");
        if (pos == std::string::npos) continue;
        const std::string base = n3.substr(0, pos), nds = base + ".0.downsample";
        auto ids = folded.find(nds);
        if (ids == folded.end()) return fail(h, -40, "missing downsample unit for " + n3);
        const ConvLayer& L3 = h->layers[n3];
        const ConvLayer& Lds = h->layers[nds];
        ConvLayer& F = h->layers[base + ".0.fused_conv3_downsample"];
        F.name = base + ".0.fused_conv3_downsample";
        F.Cin = L3.Cin;
        F.Cin2 = Lds.Cin;
        F.stride2 = Lds.stride;
        F.Cout = L3.Cout;
        F.Cout_pad = L3.Cout_pad;
        F.k = 1, F.stride = 1, F.pad = 0;
        const int cin = F.Cin + F.Cin2;
        std::vector<float> wf((size_t)F.Cout * cin), bf(F.Cout);
        for (int co = 0; co < F.Cout; co++) {
            for (int ci = 0; ci < F.Cin; ci++) wf[(size_t)co * cin + ci] = kv.second.first[(size_t)co * F.Cin + ci];
            for (int ci = 0; ci < F.Cin2; ci++)
                wf[(size_t)co * cin + F.Cin + ci] = ids->second.first[(size_t)co * F.Cin2 + ci];
            bf[co] = kv.second.second[co] + ids->second.second[co];
        }
        int rc3 = upload_conv_layer(h, F, wf, bf);
        if (rc3) return rc3;
    }
    // thin 3x3 heads as tap expansion: rows (tap*C + c) of a 1x1 GEMM, bias applied by the gather kernel
    for (auto& kv : folded) {
        const std::string& nm = kv.first;
        if (nm.find("res_d_conv2") == std::string::npos && nm.find("res_rd_conv2") == std::string::npos) continue;
        const ConvLayer& L0 = h->layers[nm];
        if (L0.k != 3) continue;
        ConvLayer& E = h->layers[nm + ".tapexp"];
        E.name = nm + ".tapexp";
        E.Cin = L0.Cin;
        E.Cout = 9 * L0.Cout;
        E.Cout_pad = pad32(E.Cout);
        E.k = 1, E.stride = 1, E.pad = 0;
        std::vector<float> wf((size_t)E.Cout * E.Cin), bf(E.Cout, 0.f);
        for (int c = 0; c < L0.Cout; c++)
            for (int ci = 0; ci < L0.Cin; ci++)
                for (int t = 0; t < 9; t++)
                    wf[(size_t)(t * L0.Cout + c) * E.Cin + ci] = kv.second.first[((size_t)c * L0.Cin + ci) * 9 + t];
        int rc4 = upload_conv_layer(h, E, wf, bf);
        if (rc4) return rc4;
    }
    if (!h->stem_w) return fail(h, -40, "top.conv weights missing");
    h->finalized = true;
    return 0;
}

int smapb_backbone_forward(smapb_handle* h, const float* imgs, int B, float* hm2d, float* detd, float* rootd,
                           void* stream) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_backbone_forward: weights not finalized");
    if (B < 1) return fail(h, -1, "B < 1");
    cudaSetDevice(h->device);
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
    if (rc) return rc;
    // NULL = legacy default stream: run on the handle's own (non-blocking) stream, bridged to the legacy stream on both sides
    if (stream) return run_plan(h, plan, imgs, hm2d, detd, rootd, (cudaStream_t)stream);
    rc = legacy_enter(h);
    if (!rc) rc = run_plan(h, plan, imgs, hm2d, detd, rootd, h->own_stream);
    if (!rc) rc = legacy_leave(h);
    return rc;
}

int smapb_merge_scale(smapb_handle* h, float* hm2d, const float* hm2d_flip, int B, int do_scale, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    CK(launch_merge_scale(hm2d, hm2d_flip, B, h->h, h->w, do_scale, (cudaStream_t)stream));
    h->launches++;
    return 0;
}

static int check_assoc(smapb_handle* h, int B) {
    if (B < 1 || B > h->max_batch) return fail(h, -1, "association: B outside [1, max_batch]");
    const char* aerr = nullptr;
    if (assoc_configure(h->h, h->w, &aerr) != 0) return fail(h, -3, aerr ? aerr : "assoc_configure failed");
    return 0;
}

int smapb_assoc_extract(smapb_handle* h, const float* hms, int B, float* peaks, float* pair_scores, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    int rc = check_assoc(h, B);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_nms(hms, NC2D, B, h->h, h->w, 0.2f, peaks, h->nms_masks, st));
    CK(launch_paf(hms, NC2D, B, h->h, h->w, peaks, pair_scores, 1, st));
    h->launches += 3;
    return 0;
}

int smapb_assoc_connect(smapb_handle* h, const float* hms, const float* rdepth, int B, int root_idx, int dist_flag,
                        float* bodies, int* counts, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    int rc = check_assoc(h, B);
    if (rc) return rc;
    if (root_idx < 0 || root_idx >= NJ) return fail(h, -1, "root_idx out of range");
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_nms(hms, NC2D, B, h->h, h->w, 0.2f, h->peaks, h->nms_masks, st));
    CK(launch_paf(hms, NC2D, B, h->h, h->w, h->peaks, h->scores, 0, st));
    CK(launch_group(h->peaks, h->scores, rdepth, B, h->h, h->w, root_idx, dist_flag, bodies, counts, st));
    h->launches += 4;
    return 0;
}

int smapb_lift3d(smapb_handle* h, const float* bodies, const int* counts, const float* detd, const float* rootd,
                 const double* scales, int B, float* pred2d, double* pred3d, double* root_depth, int* counts_out,
                 void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    if (B < 1) return fail(h, -1, "B < 1");
    CK(launch_lift(bodies, counts, detd, rootd, scales, B, h->h, h->w, 2, pred2d, pred3d, root_depth, counts_out,
                   (long long)MAXP * NJ * 4, (long long)MAXP * NJ * 4, MAXP, 1, (cudaStream_t)stream));
    h->launches++;
    return 0;
}

int smapb_lift3d_gt(smapb_handle* h, const float* bodies, const int* counts, const float* detd, const float* rootd,
                    const double* scales, const double* gt_roots, const int* gt_counts, int gmax, int B, double* pred2d,
                    double* pred3d, double* root_depth, int* counts_out, void* stream) {
    if (!h || !gt_roots || !gt_counts) return -1;
    cudaSetDevice(h->device);
    if (B < 1 || B > h->max_batch) return fail(h, -1, "smapb_lift3d_gt: B outside [1, max_batch]");
    if (gmax < 1) return fail(h, -1, "smapb_lift3d_gt: gmax < 1");
    if (!h->gt_dist && dev_alloc(h, &h->gt_dist, (size_t)h->max_batch * MAXP * MAXP)) return -10;
    CK(launch_lift_gt(bodies, counts, detd, rootd, scales, gt_roots, gt_counts, gmax, h->gt_dist, B, h->h, h->w, 2, pred2d,
                      pred3d, root_depth, counts_out, (cudaStream_t)stream));
    h->launches++;
    return 0;
}

// ---- pre-processing (SURVEY 8(f) f1) ---------------------------------------------------------------------------
static int pre_entry(smapb_handle* h, int img_h, int img_w, smapb_handle::PreEntry** out) {
    if (img_h < 2 || img_w < 2 || img_h > 16384 || img_w > 16384) return fail(h, -1, "smapb_preprocess: image size outside [2, 16384]");
    auto key = std::make_pair(img_w, img_h);
    auto it = h->pre_cache.find(key);
    if (it == h->pre_cache.end()) {
        if (h->pre_cache.size() >= 256) {  // bound the cache: drop everything (streams are idle after the sync)
            cudaDeviceSynchronize();
            for (auto& e : h->pre_cache) cudaFree(e.second.buf);
            h->pre_cache.clear();
        }
        smapb_handle::PreEntry E;
        make_resize_plan(img_w, img_h, h->in_w, h->in_h, &E.plan);
        const ResizePlan& P = E.plan;
        const size_t nx = P.xofs.size(), ny = P.yofs.size();  // ny = 2 * dst_h
        const size_t bytes = nx * 4 + ny * 4 + nx * 2 * 2 + ny * 2 + 64;
        CK(cudaMalloc(&E.buf, bytes));
        char* d = (char*)E.buf;
        int* xo = (int*)d;
        int* yo = xo + nx;
        short* xc = (short*)(yo + ny);
        short* yc = xc + 2 * nx;
        cudaError_t ce = cudaMemcpy(xo, P.xofs.data(), nx * 4, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(yo, P.yofs.data(), ny * 4, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(xc, P.xcoef.data(), nx * 2 * 2, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(yc, P.ycoef.data(), ny * 2, cudaMemcpyHostToDevice);
        if (ce != cudaSuccess) {
            cudaFree(E.buf);
            return fail(h, -10, std::string("smapb_preprocess: table upload: ") + cudaGetErrorString(ce));
        }
        E.tab = {xo, xc, yo, yc};
        it = h->pre_cache.emplace(key, std::move(E)).first;
    }
    *out = &it->second;
    return 0;
}

static void pre_scale_row(const smapb_handle* h, const ResizePlan& P, double* row) {
    if (!row) return;
    row[0] = P.scale;             // scale['scale']                    (dataset/custom_dataset.py:46)
    row[1] = P.src_w;             // img_width, img_height              (:49-50)
    row[2] = P.src_h;
    row[3] = h->in_w;             // net_width, net_height              (:51-52)
    row[4] = h->in_h;
    row[5] = P.src_w;             // f_x = f_y = img_width              (exps/stage3_root2/test.py:100-101)
    row[6] = P.src_w;
    row[7] = P.src_w / 2.0;       // cx, cy                             (test.py:102-103)
    row[8] = P.src_h / 2.0;
}

int smapb_preprocess(smapb_handle* h, const uint8_t* bgr_dev, int img_h, int img_w, float* out_nchw_dev, double* scale_row_host,
                     void* stream) {
    if (!h || !bgr_dev || !out_nchw_dev) return -1;
    cudaSetDevice(h->device);
    smapb_handle::PreEntry* E = nullptr;
    int rc = pre_entry(h, img_h, img_w, &E);
    if (rc) return rc;
    CK(launch_preprocess(bgr_dev, E->plan, E->tab, h->in_w, h->in_h, out_nchw_dev, (cudaStream_t)stream));
    h->launches++;
    pre_scale_row(h, E->plan, scale_row_host);
    return 0;
}

int smapb_preprocess_host(smapb_handle* h, const uint8_t* bgr_host, int img_h, int img_w, float* out_nchw_dev,
                          double* scale_row_host, void* stream) {
    if (!h || !bgr_host || !out_nchw_dev) return -1;
    cudaSetDevice(h->device);
    const size_t bytes = (size_t)img_h * img_w * 3;
    if (bytes > h->pre_stage_bytes) {
        cudaDeviceSynchronize();
        if (h->pre_stage) cudaFree(h->pre_stage);
        h->pre_stage = nullptr;
        h->pre_stage_bytes = 0;
        CK(cudaMalloc((void**)&h->pre_stage, bytes));
        h->pre_stage_bytes = bytes;
    }
    CK(cudaMemcpyAsync(h->pre_stage, bgr_host, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return smapb_preprocess(h, h->pre_stage, img_h, img_w, out_nchw_dev, scale_row_host, stream);
}

// host-only introspection of the resampling plan (tests compare it with the oracle over many geometries without a GPU)
int smapb_debug_resize_plan(int src_w, int src_h, int net_w, int net_h, int* dims6, double* scale, int* xofs, short* xcoef,
                            int* yofs, short* ycoef) {
    if (src_w < 2 || src_h < 2 || net_w < 1 || net_h < 1 || !dims6) return -1;
    ResizePlan P;
    make_resize_plan(src_w, src_h, net_w, net_h, &P);
    dims6[0] = P.dst_w, dims6[1] = P.dst_h, dims6[2] = P.pad_l, dims6[3] = P.pad_t, dims6[4] = P.mode, dims6[5] = 0;
    if (scale) *scale = P.scale;
    if (xofs) memcpy(xofs, P.xofs.data(), P.xofs.size() * sizeof(int));
    if (xcoef) memcpy(xcoef, P.xcoef.data(), P.xcoef.size() * sizeof(short));
    if (yofs) memcpy(yofs, P.yofs.data(), P.yofs.size() * sizeof(int));
    if (ycoef) memcpy(ycoef, P.ycoef.data(), P.ycoef.size() * sizeof(short));
    return 0;
}

// ---- RefineNet (SURVEY 8(f) f2) ---------------------------------------------------------------------------------
int smapb_refine_load_weight(smapb_handle* h, const char* key, const float* host, const int64_t* shape, int ndim) {
    if (!h || !key || !host) return -1;
    const std::string k(key);
    if (k.size() > 19 && k.compare(k.size() - 19, 19, "num_batches_tracked") == 0) return 0;
    size_t n = 1;
    for (int i = 0; i < ndim; i++) n *= (size_t)shape[i];
    h->refine_raw[k].assign(host, host + n);
    h->refine_ready = false;
    return 0;
}

int smapb_refine_finalize(smapb_handle* h) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    static const int dims[RF_LAYERS + 1] = {75, 160, 256, 256, 128, 45};
    size_t total = 0;
    for (int l = 0; l < RF_LAYERS; l++) total += (size_t)dims[l] * dims[l + 1] + dims[l + 1];
    std::vector<float> buf(total);
    size_t off = 0, w_off[RF_LAYERS], b_off[RF_LAYERS];
    for (int l = 0; l < RF_LAYERS; l++) {
        const int K = dims[l], N = dims[l + 1];
        const bool has_bn = l < RF_LAYERS - 1;
        const std::string lp = "block.layer" + std::to_string(l + 1) + (has_bn ? ".0." : ".");
        const std::string bp = "block.layer" + std::to_string(l + 1) + ".1.";
        auto get = [&](const std::string& key, size_t n, const std::vector<float>** out) -> int {
            auto it = h->refine_raw.find(key);
            if (it == h->refine_raw.end()) return fail(h, -3, "smapb_refine_finalize: missing key " + key);
            if (it->second.size() != n) return fail(h, -3, "smapb_refine_finalize: wrong size for " + key);
            *out = &it->second;
            return 0;
        };
        const std::vector<float>*w = nullptr, *b = nullptr, *g = nullptr, *be = nullptr, *mu = nullptr, *var = nullptr;
        int rc = get(lp + "weight", (size_t)K * N, &w);
        if (!rc) rc = get(lp + "bias", N, &b);
        if (!rc && has_bn) rc = get(bp + "weight", N, &g);
        if (!rc && has_bn) rc = get(bp + "bias", N, &be);
        if (!rc && has_bn) rc = get(bp + "running_mean", N, &mu);
        if (!rc && has_bn) rc = get(bp + "running_var", N, &var);
        if (rc) return rc;
        w_off[l] = off;
        b_off[l] = off + (size_t)K * N;
        for (int n = 0; n < N; n++) {
            // BatchNorm1d(eval), eps 1e-5 (model/refinenet.py:9): y = (Wx + b - mu) * g / sqrt(var + eps) + beta
            const double sc = has_bn ? (double)(*g)[n] / sqrt((double)(*var)[n] + 1e-5) : 1.0;
            for (int k = 0; k < K; k++) buf[w_off[l] + (size_t)k * N + n] = (float)((double)(*w)[(size_t)n * K + k] * sc);
            buf[b_off[l] + n] = has_bn ? (float)(((double)(*b)[n] - (double)(*mu)[n]) * sc + (double)(*be)[n]) : (*b)[n];
        }
        off += (size_t)K * N + N;
    }
    if (!h->refine_buf) CK(cudaMalloc((void**)&h->refine_buf, total * sizeof(float)));
    CK(cudaMemcpy(h->refine_buf, buf.data(), total * sizeof(float), cudaMemcpyHostToDevice));
    for (int l = 0; l < RF_LAYERS; l++) {
        h->refine_w.w[l] = h->refine_buf + w_off[l];
        h->refine_w.b[l] = h->refine_buf + b_off[l];
    }
    h->refine_ready = true;
    return 0;
}

int smapb_set_refine(smapb_handle* h, int enable) {
    if (!h) return -1;
    if (enable && !h->refine_ready) return fail(h, -2, "smapb_set_refine: RefineNet weights not finalized");
    if ((enable != 0) != h->refine_on) {  // captured graphs contain (or lack) the refine launch
        cudaSetDevice(h->device);
        cudaDeviceSynchronize();
        for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
        h->graphs.clear();
    }
    h->refine_on = enable != 0;
    return 0;
}

int smapb_refine_mlp(smapb_handle* h, const float* in_dev, int n, float* out_dev, void* stream) {
    if (!h) return -1;
    if (!h->refine_ready) return fail(h, -2, "smapb_refine_mlp: RefineNet weights not finalized");
    if (n < 0) return fail(h, -1, "smapb_refine_mlp: n < 0");
    cudaSetDevice(h->device);
    CK(launch_refine_mlp(h->refine_w, in_dev, n, out_dev, (cudaStream_t)stream));
    if (n) h->launches++;
    return 0;
}

int smapb_refine3d(smapb_handle* h, const float* pred2d, const double* pred3d, const int* counts, int B, int root_idx,
                   double* refined, void* stream) {
    if (!h) return -1;
    if (!h->refine_ready) return fail(h, -2, "smapb_refine3d: RefineNet weights not finalized");
    if (B < 1) return fail(h, -1, "B < 1");
    if (root_idx < 0 || root_idx >= NJ) return fail(h, -1, "root_idx outside [0, 15)");
    cudaSetDevice(h->device);
    CK(launch_refine_records(h->refine_w, pred2d, pred3d, counts, B, root_idx, (long long)MAXP * NJ * 4, (long long)MAXP * NJ * 4,
                             1, refined, (long long)MAXP * NJ * 4, (cudaStream_t)stream));
    h->launches++;
    return 0;
}

// flip along W of an NCHW fp32 batch (torch.flip(imgs, [-1]), exps/stage3_root2/test.py:56)
__global__ void flip_w_kernel(const float* __restrict__ in, float* __restrict__ out, long long rows, int W) {
    const long long total = rows * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / W;
        const int x = (int)(i - r * W);
        out[i] = in[r * W + (W - 1 - x)];
    }
}

static int infer_body(smapb_handle* h, Plan* plan, const float* imgs, const double* scales, int B, int do_flip,
                      smapb_record* records, cudaStream_t st) {
    nvtxRangePushA("smapb.backbone");
    int rc = run_plan(h, plan, imgs, h->hm, h->detd, h->rootd, st);
    if (rc) {
        nvtxRangePop();
        return rc;
    }
    const size_t hw = (size_t)h->h * h->w;
    if (do_flip) {
        const size_t MB = h->max_batch;
        if (!h->imgs_flip) {
            if (dev_alloc(h, &h->imgs_flip, MB * 3 * h->in_h * h->in_w)) return -10;
            if (dev_alloc(h, &h->hm_flip, MB * NC2D * hw)) return -10;
            if (dev_alloc(h, &h->scratch_detd, MB * NL * hw)) return -10;
            if (dev_alloc(h, &h->scratch_rootd, MB * hw)) return -10;
        }
        flip_w_kernel<<<132 * 8, 256, 0, st>>>(imgs, h->imgs_flip, (long long)B * 3 * h->in_h, h->in_w);
        CK(cudaGetLastError());
        prof_mark(h, PK_ELEM, st, "flip_w");
        h->launches++;
        rc = run_plan(h, plan, h->imgs_flip, h->hm_flip, h->scratch_detd, h->scratch_rootd, st);
        if (rc) {
            nvtxRangePop();
            return rc;
        }
    }
    nvtxRangePop();
    nvtxRangePushA("smapb.association");
    CK(launch_merge_scale(h->hm, do_flip ? h->hm_flip : nullptr, B, h->h, h->w, 1, st));
    prof_mark(h, PK_ELEM, st, "merge_scale");
    CK(launch_nms(h->hm, NC2D, B, h->h, h->w, 0.2f, h->peaks, h->nms_masks, st));
    prof_mark(h, PK_ASSOC, st, "nms");
    CK(launch_paf(h->hm, NC2D, B, h->h, h->w, h->peaks, h->scores, 0, st));
    prof_mark(h, PK_ASSOC, st, "paf");
    CK(launch_group(h->peaks, h->scores, h->rootd, B, h->h, h->w, 2, 1, h->bodies, h->counts, st));
    prof_mark(h, PK_ASSOC, st, "group");
    nvtxRangePop();
    nvtxRangePushA("smapb.lift");
    char* rb = reinterpret_cast<char*>(records);
    CK(launch_lift(h->bodies, h->counts, h->detd, h->rootd, scales, B, h->h, h->w, 2,
                   reinterpret_cast<float*>(rb + offsetof(smapb_record, pred2d)),
                   reinterpret_cast<double*>(rb + offsetof(smapb_record, pred3d)),
                   reinterpret_cast<double*>(rb + offsetof(smapb_record, root_depth)),
                   reinterpret_cast<int*>(rb + offsetof(smapb_record, count)), sizeof(smapb_record) / 4,
                   sizeof(smapb_record) / 8, sizeof(smapb_record) / 8, sizeof(smapb_record) / 4, st));
    prof_mark(h, PK_LIFT, st, "lift");
    h->launches += 6;
    if (h->refine_on) {  // refined poses replace pred3d, as save_result(pred_bodys_2d, new_pred_bodys_3d, ...) does (test.py:137-145)
        double* p3 = reinterpret_cast<double*>(rb + offsetof(smapb_record, pred3d));
        CK(launch_refine_records(h->refine_w, reinterpret_cast<float*>(rb + offsetof(smapb_record, pred2d)), p3,
                                 reinterpret_cast<int*>(rb + offsetof(smapb_record, count)), B, 2, sizeof(smapb_record) / 4,
                                 sizeof(smapb_record) / 8, sizeof(smapb_record) / 4, p3, sizeof(smapb_record) / 8, st));
        prof_mark(h, PK_LIFT, st, "refine");
        h->launches++;
    }
    nvtxRangePop();
    return 0;
}

// one all-gather of B fixed-stride records per rank (SURVEY 8(e)), on `st`
static int gather_records(smapb_handle* h, void* comm, const smapb_record* send, smapb_record* recv, int B, cudaStream_t st) {
    NcclApi& a = nccl_api();
    if (!a.lib) return fail(h, -51, a.err.empty() ? "NCCL unavailable" : a.err);
    if (!comm) return fail(h, -52, "no NCCL communicator");
    const int rc = a.AllGather(send, recv, (size_t)B * sizeof(smapb_record), /* ncclUint8 */ 1, comm, st);
    if (rc != 0) return nccl_fail(h, "ncclAllGather", rc);
    return 0;
}

// Whole path on stream `st` (never NULL here).  gather != 0: followed by the all-gather of the records over the handle's
// communicator; `records` then receives comm_world * B records in rank order.
static int infer_device_impl(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip, int gather,
                             smapb_record* records, cudaStream_t st) {
    int rc = check_assoc(h, B);
    if (rc) return rc;
    if (gather && !h->comm) return fail(h, -52, "smapb_infer_*_gather: no communicator attached (smapb_comm_create / smapb_comm_attach)");
    if (gather && !h->gather_dev) return fail(h, -52, "gather buffer missing");
    Plan* plan = nullptr;
    rc = build_plan(h, B, &plan);
    if (rc) return rc;
    do_flip = do_flip ? 1 : 0;
    gather = gather ? 1 : 0;
    const size_t out_records = (size_t)B * (gather ? h->comm_world : 1);
    static const bool no_graph = getenv("SMAPB_NO_GRAPH") != nullptr;
    // The whole path (~210 launches) is replayed from a CUDA graph: the first two calls for a (B, flip, gather) run
    // eagerly (lazy allocations, function attributes, NCCL connection setup), then one graph per distinct input pointer
    // pair is captured - with the all-gather inside when NCCL accepts the capture.  Results land in handle-owned
    // buffers and are copied to the caller's pointer behind the graph.
    int& eager = h->eager_runs[{B, do_flip * 2 + gather}];
    if (no_graph || h->profiling || eager < 2) {
        eager++;
        if (!gather) return infer_body(h, plan, imgs, scales, B, do_flip, records, st);
        rc = infer_body(h, plan, imgs, scales, B, do_flip, h->records_dev, st);
        if (rc) return rc;
        return gather_records(h, h->comm, h->records_dev, records, B, st);
    }
    smapb_handle::GraphEntry* ge = nullptr;
    for (auto& g : h->graphs)
        if (g.B == B && g.flip == do_flip && g.gather == gather && g.imgs == imgs && g.scales == scales) ge = &g;
    const bool gather_in_graph = gather && h->nccl_in_graph;
    if (!ge) {
        if (h->graphs.size() >= 16) {  // evict the least recently used graph (callers that pass ever-changing pointers)
            size_t lru = 0;
            for (size_t i = 1; i < h->graphs.size(); i++)
                if (h->graphs[i].stamp < h->graphs[lru].stamp) lru = i;
            cudaGraphExecDestroy(h->graphs[lru].exec);
            h->graphs.erase(h->graphs.begin() + lru);
        }
        const int64_t launches_before = h->launches;
        CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        rc = infer_body(h, plan, imgs, scales, B, do_flip, h->records_dev, st);
        if (!rc && gather_in_graph) rc = gather_records(h, h->comm, h->records_dev, h->gather_dev, B, st);
        cudaGraph_t graph = nullptr;
        cudaError_t ce = cudaStreamEndCapture(st, &graph);
        h->launches = launches_before;
        if (rc) {
            if (graph) cudaGraphDestroy(graph);
            return rc;
        }
        if (ce != cudaSuccess) return fail(h, -10, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
        cudaGraphExec_t exec = nullptr;
        ce = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ce != cudaSuccess) return fail(h, -10, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce));
        h->graphs.push_back({B, do_flip, gather, imgs, scales, exec, 0});
        ge = &h->graphs.back();
    }
    ge->stamp = ++h->graph_clock;
    CK(cudaGraphLaunch(ge->exec, st));
    h->launches += (int64_t)plan->ops.size() * (do_flip ? 2 : 1) + 6 + (do_flip ? 1 : 0) + (h->refine_on ? 1 : 0);
    const smapb_record* src = h->records_dev;
    if (gather) {
        if (!gather_in_graph) {  // NCCL outside the graph, still stream-ordered on the compute stream
            rc = gather_records(h, h->comm, h->records_dev, h->gather_dev, B, st);
            if (rc) return rc;
        }
        src = h->gather_dev;
    }
    if (records != src)
        CK(cudaMemcpyAsync(records, src, out_records * sizeof(smapb_record), cudaMemcpyDeviceToDevice, st));
    return 0;
}

static int gather_side_init(smapb_handle* h) {
    if (h->gather_stream) return 0;
    CK(cudaStreamCreateWithFlags(&h->gather_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) {
        CK(cudaEventCreateWithFlags(&h->rec_ready[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->gather_done[i], cudaEventDisableTiming));
        if (dev_alloc(h, &h->rec_buf[i], (size_t)h->max_batch)) return -10;
    }
    return 0;
}

// Whole path on `st`, exchange on the handle's gather stream: `st` is ordered after the COMPUTE only.  all_records is valid
// once smapb_gather_sync has made a stream wait for the exchange.  The records are double-buffered, so a call only waits for
// the exchange issued two calls earlier.
static int infer_device_gather_async_impl(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                                          smapb_record* all_records, cudaStream_t st) {
    if (!h->comm) return fail(h, -52, "smapb_infer_device_gather_async: no communicator attached");
    int rc = gather_side_init(h);
    if (rc) return rc;
    const int idx = h->gather_idx;
    h->gather_idx ^= 1;
    if (h->gather_used[idx]) CK(cudaStreamWaitEvent(st, h->gather_done[idx], 0));
    rc = infer_device_impl(h, imgs, scales, B, do_flip, 0, h->rec_buf[idx], st);
    if (rc) return rc;
    CK(cudaEventRecord(h->rec_ready[idx], st));
    CK(cudaStreamWaitEvent(h->gather_stream, h->rec_ready[idx], 0));
    rc = gather_records(h, h->comm, h->rec_buf[idx], all_records, B, h->gather_stream);
    if (rc) return rc;
    CK(cudaEventRecord(h->gather_done[idx], h->gather_stream));
    h->gather_used[idx] = true;
    return 0;
}

static int infer_device_entry(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip, int gather,
                              smapb_record* records, void* stream) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_infer_device: weights not finalized");
    cudaSetDevice(h->device);
    if (stream) return infer_device_impl(h, imgs, scales, B, do_flip, gather, records, (cudaStream_t)stream);
    // The legacy default stream cannot be captured: run on the handle's own stream, bridged on both sides
    int rc = legacy_enter(h);
    if (!rc) rc = infer_device_impl(h, imgs, scales, B, do_flip, gather, records, h->own_stream);
    if (!rc) rc = legacy_leave(h);
    return rc;
}

int smapb_infer_device(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                       smapb_record* records, void* stream) {
    return infer_device_entry(h, imgs, scales, B, do_flip, 0, records, stream);
}

int smapb_infer_device_gather(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                              smapb_record* all_records, void* stream) {
    return infer_device_entry(h, imgs, scales, B, do_flip, 1, all_records, stream);
}

int smapb_infer_device_gather_async(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                                    smapb_record* all_records, void* stream) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_infer_device_gather_async: weights not finalized");
    cudaSetDevice(h->device);
    if (stream) return infer_device_gather_async_impl(h, imgs, scales, B, do_flip, all_records, (cudaStream_t)stream);
    int rc = legacy_enter(h);
    if (!rc) rc = infer_device_gather_async_impl(h, imgs, scales, B, do_flip, all_records, h->own_stream);
    if (!rc) rc = legacy_leave(h);
    return rc;
}

int smapb_gather_sync(smapb_handle* h, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    cudaStream_t st = stream ? (cudaStream_t)stream : cudaStreamLegacy;
    for (int i = 0; i < 2; i++)
        if (h->gather_used[i]) CK(cudaStreamWaitEvent(st, h->gather_done[i], 0));
    return 0;
}

int smapb_infer_host(smapb_handle* h, const float* imgs_host, const double* scales_host, int B, int do_flip,
                     smapb_record* records_host, void* stream) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_infer_host: weights not finalized");
    if (B < 1 || B > h->max_batch) return fail(h, -1, "smapb_infer_host: B outside [1, max_batch]");
    cudaSetDevice(h->device);
    cudaStream_t st = stream ? (cudaStream_t)stream : h->own_stream;
    if (!stream) {
        int rc0 = legacy_enter(h);
        if (rc0) return rc0;
    }
    CK(cudaMemcpyAsync(h->imgs_dev, imgs_host, (size_t)B * 3 * h->in_h * h->in_w * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->scales_dev, scales_host, (size_t)B * SMAPB_SCALE_LEN * 8, cudaMemcpyHostToDevice, st));
    int rc = infer_device_impl(h, h->imgs_dev, h->scales_dev, B, do_flip, 0, h->records_dev, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(records_host, h->records_dev, (size_t)B * sizeof(smapb_record), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

static int submit_host_impl(smapb_handle* h, int slot, const float* imgs_host, const double* scales_host, int B, int do_flip,
                            int gather, smapb_record* records_host) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_submit_host: weights not finalized");
    if (slot < 0 || slot > 1) return fail(h, -1, "smapb_submit_host: slot must be 0 or 1");
    if (B < 1 || B > h->max_batch) return fail(h, -1, "smapb_submit_host: B outside [1, max_batch]");
    if (gather && !h->comm) return fail(h, -52, "smapb_submit_host_gather: no communicator attached");
    cudaSetDevice(h->device);
    smapb_handle::Slot& S = h->slots[slot];
    if (!S.imgs) {
        const size_t MB = h->max_batch;
        if (dev_alloc(h, &S.imgs, MB * 3 * h->in_h * h->in_w)) return -10;
        if (dev_alloc(h, &S.scales, MB * SMAPB_SCALE_LEN)) return -10;
        if (dev_alloc(h, &S.records, MB)) return -10;
        CK(cudaEventCreateWithFlags(&S.h2d, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&S.done, cudaEventDisableTiming));
        if (!h->copy_stream) CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    }
    if (gather && !S.records_all && dev_alloc(h, &S.records_all, (size_t)h->max_batch * h->comm_world)) return -10;
    // the slot's buffers are free once its previous submission has completed
    if (S.used) CK(cudaStreamWaitEvent(h->copy_stream, S.done, 0));
    CK(cudaMemcpyAsync(S.imgs, imgs_host, (size_t)B * 3 * h->in_h * h->in_w * 4, cudaMemcpyHostToDevice, h->copy_stream));
    CK(cudaMemcpyAsync(S.scales, scales_host, (size_t)B * SMAPB_SCALE_LEN * 8, cudaMemcpyHostToDevice, h->copy_stream));
    CK(cudaEventRecord(S.h2d, h->copy_stream));
    cudaStream_t st = h->own_stream;
    CK(cudaStreamWaitEvent(st, S.h2d, 0));
    int rc = infer_device_impl(h, S.imgs, S.scales, B, do_flip, 0, S.records, st);
    if (rc) return rc;
    if (!gather) {
        CK(cudaMemcpyAsync(records_host, S.records, (size_t)B * sizeof(smapb_record), cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(S.done, st));
    } else {
        // The exchange and the D2H of its result run on the gather stream: the compute stream goes straight on to the next
        // slot's batch and never waits for a peer.  The records are exchanged on the device (NVLink) and leave in ONE D2H -
        // nothing is re-uploaded.
        rc = gather_side_init(h);
        if (rc) return rc;
        if (!S.rec_ready) CK(cudaEventCreateWithFlags(&S.rec_ready, cudaEventDisableTiming));
        CK(cudaEventRecord(S.rec_ready, st));
        CK(cudaStreamWaitEvent(h->gather_stream, S.rec_ready, 0));
        rc = gather_records(h, h->comm, S.records, S.records_all, B, h->gather_stream);
        if (rc) return rc;
        CK(cudaMemcpyAsync(records_host, S.records_all, (size_t)B * h->comm_world * sizeof(smapb_record), cudaMemcpyDeviceToHost,
                           h->gather_stream));
        CK(cudaEventRecord(S.done, h->gather_stream));
    }
    S.used = true;
    return 0;
}

int smapb_submit_host(smapb_handle* h, int slot, const float* imgs_host, const double* scales_host, int B, int do_flip,
                      smapb_record* records_host) {
    return submit_host_impl(h, slot, imgs_host, scales_host, B, do_flip, 0, records_host);
}

int smapb_submit_host_gather(smapb_handle* h, int slot, const float* imgs_host, const double* scales_host, int B, int do_flip,
                             smapb_record* all_records_host) {
    return submit_host_impl(h, slot, imgs_host, scales_host, B, do_flip, 1, all_records_host);
}

int smapb_wait(smapb_handle* h, int slot) {
    if (!h) return -1;
    if (slot < 0 || slot > 1 || !h->slots[slot].used) return fail(h, -1, "smapb_wait: nothing submitted on this slot");
    cudaSetDevice(h->device);
    CK(cudaEventSynchronize(h->slots[slot].done));
    return 0;
}

// ---- multi-GPU: communicator + the one exchange step of the path (SURVEY 8(e)) ----------------------------------
int smapb_comm_unique_id(void* id128) {
    NcclApi& a = nccl_api();
    if (!a.lib || !id128) return -51;
    NcclUid id;
    const int rc = a.GetUniqueId(&id);
    if (rc != 0) return -50;
    memcpy(id128, &id, 128);
    return 0;
}

static int set_comm(smapb_handle* h, void* comm, bool owned, int rank, int world) {
    if (world < 1 || rank < 0 || rank >= world) return fail(h, -1, "communicator: rank / world out of range");
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    if (h->comm && h->comm_owned && nccl_api().CommDestroy) nccl_api().CommDestroy(h->comm);
    // graphs captured with the previous communicator (or without one) stay valid only for gather == 0
    for (size_t i = 0; i < h->graphs.size();) {
        if (h->graphs[i].gather) {
            cudaGraphExecDestroy(h->graphs[i].exec);
            h->graphs.erase(h->graphs.begin() + i);
        } else {
            i++;
        }
    }
    for (auto& kv : h->eager_runs)
        if (kv.first.second & 1) kv.second = 0;
    h->comm = comm, h->comm_owned = owned, h->comm_rank = rank, h->comm_world = world;
    if (h->gather_dev) cudaFree(h->gather_dev);
    h->gather_dev = nullptr;
    for (auto& S : h->slots) {
        cudaFree(S.records_all);
        S.records_all = nullptr;
    }
    if (dev_alloc(h, &h->gather_dev, (size_t)world * h->max_batch)) return -10;
    return 0;
}

int smapb_comm_create(smapb_handle* h, const void* id128, int rank, int world) {
    if (!h || !id128) return -1;
    NcclApi& a = nccl_api();
    if (!a.lib) return fail(h, -51, a.err.empty() ? "NCCL unavailable" : a.err);
    cudaSetDevice(h->device);
    NcclUid id;
    memcpy(&id, id128, 128);
    void* comm = nullptr;
    const int rc = a.CommInitRank(&comm, world, id, rank);
    if (rc != 0) return nccl_fail(h, "ncclCommInitRank", rc);
    return set_comm(h, comm, true, rank, world);
}

int smapb_comm_attach(smapb_handle* h, void* nccl_comm, int rank, int world) {
    if (!h || !nccl_comm) return -1;
    NcclApi& a = nccl_api();
    if (!a.lib) return fail(h, -51, a.err.empty() ? "NCCL unavailable" : a.err);
    return set_comm(h, nccl_comm, false, rank, world);
}

int smapb_allgather_records(smapb_handle* h, void* nccl_comm, const smapb_record* records_dev, smapb_record* all_records_dev,
                            int B, void* stream) {
    if (!h || !records_dev || !all_records_dev) return -1;
    if (B < 1) return fail(h, -1, "smapb_allgather_records: B < 1");
    cudaSetDevice(h->device);
    void* comm = nccl_comm ? nccl_comm : h->comm;
    if (stream) return gather_records(h, comm, records_dev, all_records_dev, B, (cudaStream_t)stream);
    int rc = legacy_enter(h);
    if (!rc) rc = gather_records(h, comm, records_dev, all_records_dev, B, h->own_stream);
    if (!rc) rc = legacy_leave(h);
    return rc;
}

// ---- tile-shape table (process-wide) ------------------------------------------------------------------------------
int smapb_set_tile_table(const char* text) {
    if (!text) return -1;
    std::lock_guard<std::mutex> lk(g_tiles_mu);
    int n = 0;
    const char* p = text;
    while (*p) {
        const char* e = strchr(p, '\n');
        std::string line = e ? std::string(p, e - p) : std::string(p);
        p = e ? e + 1 : p + line.size();
        if (line.empty() || line[0] == '#') continue;
        const size_t t1 = line.find('\t');
        if (t1 == std::string::npos) continue;
        int bn = 0, cg = 1;
        if (sscanf(line.c_str() + t1 + 1, "%d\t%d", &bn, &cg) < 1 || bn <= 0) continue;
        g_tiles[line.substr(0, t1)] = {bn, cg};
        n++;
    }
    return n;
}

int smapb_get_tile_table(char* buf, int cap) {
    std::lock_guard<std::mutex> lk(g_tiles_mu);
    std::string out;
    for (auto& kv : g_tiles) out += kv.first + "\t" + std::to_string(kv.second.first) + "\t" + std::to_string(kv.second.second) + "\n";
    if (buf && cap > 0) {
        const size_t n = std::min((size_t)cap - 1, out.size());
        memcpy(buf, out.data(), n);
        buf[n] = 0;
    }
    return (int)out.size() + 1;
}

// debug: 64-bit checksums of every plan op's output tensor after the last forward (tools/debug_ops.py)
__global__ void checksum_kernel(const uint32_t* __restrict__ p, long long nwords, unsigned long long* out) {
    unsigned long long acc = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (long long)gridDim.x * blockDim.x)
        acc += (unsigned long long)p[i] * (unsigned long long)((i % 1021) + 1);
    atomicAdd(out, acc);
}
// debug: raw copy of plan op `idx`'s split output (both planes, bf16 bits) to host; returns bytes copied
long long smapb_debug_dump(smapb_handle* h, int B, int idx, void* host, long long max_bytes, int which) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
    if (rc) return rc;
    cudaDeviceSynchronize();
    int n = 0;
    for (const Op& op : plan->ops) {
        long long bytes = 0;
        const void* ptr = dumped_output(h, op, &bytes);
        if (!ptr) continue;
        if (n++ != idx) continue;
        (void)which;
        if (bytes > max_bytes) bytes = max_bytes;
        // cudaMemcpyDefault: `host` may also be device memory (a test keeps large dumps on the GPU)
        if (bytes > 0) CK(cudaMemcpy(host, ptr, (size_t)bytes, cudaMemcpyDefault));
        return bytes;
    }
    return -2;
}

int smapb_debug_checksums(smapb_handle* h, int B, unsigned long long* sums, int max_ops, char* desc, int desc_stride) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
    if (rc) return rc;
    CK(cudaDeviceSynchronize());
    unsigned long long* d = nullptr;
    CK(cudaMalloc((void**)&d, 8));
    std::map<const void*, int> dump_idx;  // output tensor -> dump index (the numbering of smapb_debug_dump)
    int n_dumped = 0;
    for (const Op& op : plan->ops) {
        long long bytes = 0;
        const void* out = dumped_output(h, op, &bytes);
        if (!out) continue;
        if (!dump_idx.emplace(out, n_dumped++).second) {
            cudaFree(d);
            return fail(h, -2, "smapb_debug_checksums: two ops share an output tensor (" + op.name + ")");
        }
    }
    int n = 0;
    for (const Op& op : plan->ops) {
        if (n >= max_ops) break;
        long long bytes = 0;
        const void* ptr = dumped_output(h, op, &bytes);
        if (!ptr) continue;
        const long long words = bytes / 4;
        CK(cudaMemset(d, 0, 8));
        checksum_kernel<<<132 * 4, 256>>>((const uint32_t*)ptr, words, d);
        CK(cudaMemcpy(&sums[n], d, 8, cudaMemcpyDeviceToHost));
        if (desc) snprintf(desc + (size_t)n * desc_stride, desc_stride, "%s", debug_op_desc(h, op, dump_idx).c_str());
        n++;
    }
    cudaFree(d);
    return n;
}

int64_t smapb_launch_count(const smapb_handle* h) { return h ? h->launches : 0; }

int64_t smapb_saturation_count(smapb_handle* h, int reset) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    CK(cudaDeviceSynchronize());  // the handle's work runs on non-blocking streams
    unsigned long long n = 0;
    CK(cudaMemcpy(&n, h->sat_dev, sizeof n, cudaMemcpyDeviceToHost));
    if (reset) CK(cudaMemset(h->sat_dev, 0, sizeof n));
    return (int64_t)n;
}

int smapb_profile_begin(smapb_handle* h) {
    if (!h) return -1;
    h->profiling = true;
    h->prof_used = 0;
    if (getenv("SMAPB_ROLES_PLAN")) {
        cudaSetDevice(h->device);
        if (!h->roles_dev) CK(cudaMalloc((void**)&h->roles_dev, ROLES_CAP * 16 * sizeof(long long)));
        CK(cudaMemset(h->roles_dev, 0, ROLES_CAP * 16 * sizeof(long long)));
        h->roles_used = 0;
        h->roles_desc.clear();
    }
    return 0;
}

int smapb_profile_end(smapb_handle* h, double* ms_by_kind, int* launches_by_kind, const char* csv_path) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    h->profiling = false;
    CK(cudaDeviceSynchronize());
    for (int k = 0; k < 6; k++) {
        if (ms_by_kind) ms_by_kind[k] = 0;
        if (launches_by_kind) launches_by_kind[k] = 0;
    }
    FILE* f = csv_path ? fopen(csv_path, "w") : nullptr;
    if (f) fprintf(f, "idx,kind,ms,gflop,tflops,desc\n");
    for (size_t i = 1; i < h->prof_used; i++) {
        const int k = h->prof_kind[i];
        if (k < 0) continue;
        float ms = 0;
        cudaEventElapsedTime(&ms, h->prof_events[i - 1], h->prof_events[i]);
        if (ms_by_kind) ms_by_kind[k] += ms;
        if (launches_by_kind) launches_by_kind[k]++;
        if (f)
            fprintf(f, "%zu,%d,%.5f,%.4f,%.2f,%s\n", i, k, ms, h->prof_flops[i] * 1e-9,
                    ms > 0 ? h->prof_flops[i] / (ms * 1e-3) * 1e-12 : 0.0, h->prof_desc[i].c_str());
    }
    if (f) fclose(f);
    h->prof_used = 0;
    if (h->roles_dev && h->roles_used && getenv("SMAPB_ROLES_PLAN")) {
        // mean cycles per role and CTA of every conv launch of the profiled window (counter layout: ConvDbg)
        std::vector<long long> d(h->roles_used * 16);
        CK(cudaMemcpy(d.data(), h->roles_dev, d.size() * sizeof(long long), cudaMemcpyDeviceToHost));
        FILE* g = fopen(getenv("SMAPB_ROLES_PLAN"), "w");
        if (g) {
            fprintf(g, "idx,name,desc,ctas,total,producer_wait_empty,g0_wait_full,g0_wait_order,g0_epilogue,g0_wait_ring,"
                       "g0_wait_stage,g1_wait_full,g1_wait_order,g1_epilogue,g1_wait_ring,g1_wait_stage\n");
            for (size_t i = 0; i < h->roles_used && i < h->roles_desc.size(); i++) {
                const long long* r = &d[i * 16];
                const double n = r[ConvDbg::CTAS] > 0 ? (double)r[ConvDbg::CTAS] : 1.0;
                fprintf(g, "%zu,%s,%.0f,%.0f,%.0f", i, h->roles_desc[i].c_str(), n, r[ConvDbg::TOTAL] / n,
                        r[ConvDbg::PRODUCER_WAIT_EMPTY] / n);
                for (int c = ConvDbg::CONS; c < ConvDbg::COUNT; c++) fprintf(g, ",%.0f", r[c] / n);
                fprintf(g, "\n");
            }
            fclose(g);
        }
        h->roles_used = 0;
    }
    return 0;
}

int smapb_plan_info(const smapb_handle* hc, int B, int* n_conv, double* conv_flops) {
    smapb_handle* h = const_cast<smapb_handle*>(hc);
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "weights not finalized");
    cudaSetDevice(h->device);
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
    if (rc) return rc;
    if (n_conv) *n_conv = plan->n_conv;
    if (conv_flops) *conv_flops = plan->conv_flops;
    return 0;
}

// split-bf16 planes (or the fp16 plane, f16 != 0) -> fp32 (test hook)
__global__ void split_to_f32_kernel(const __nv_bfloat16* __restrict__ in, long long plane, int terms, float* __restrict__ out,
                                    long long n, int f16) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (f16) {
        out[i] = __half2float(reinterpret_cast<const __half*>(in)[i]);
        return;
    }
    float v = __bfloat162float(in[i]);
    if (terms == 2) v += __bfloat162float(in[plane + i]);
    out[i] = v;
}

int smapb_conv_test(smapb_handle* h, const float* x, const float* w, const float* bias, const float* res,
                    const float* post1, const float* post2, int B, int H, int W, int Cin, int Cout, int k, int stride,
                    int relu, int precision, float* y, float* ms_out, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (precision != SMAPB_PREC_BF16X3 && precision != SMAPB_PREC_BF16 && precision != SMAPB_PREC_FP16)
        return fail(h, -1, "smapb_conv_test: unknown precision");
    const int save_terms = h->nterms, save_planes = h->planes;
    const bool save_f16 = h->f16;
    h->nterms = precision == SMAPB_PREC_BF16X3 ? 3 : 1;
    h->planes = precision == SMAPB_PREC_BF16X3 ? 2 : 1;
    h->f16 = precision == SMAPB_PREC_FP16;
    int rc = 0;
    ConvLayer L;
    L.name = "conv_test";
    L.Cin = Cin, L.Cout = Cout, L.Cout_pad = pad32(Cout), L.k = k, L.stride = stride, L.pad = k / 2, L.relu = relu;
    std::vector<float> wh((size_t)Cout * Cin * k * k), bh(Cout);
    std::vector<void*> tmp;
    auto cleanup = [&]() {
        for (void* p : tmp) cudaFree(p);
        cudaFree(L.w_dev);
        cudaFree(L.bias_dev);
        h->nterms = save_terms;
        h->planes = save_planes;
        h->f16 = save_f16;
    };
#define CKT(call)                                                                         \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess) {                                                          \
            cleanup();                                                                    \
            return fail(h, -10, std::string(#call) + ": " + cudaGetErrorString(e_));      \
        }                                                                                 \
    } while (0)
    CKT(cudaMemcpy(wh.data(), w, wh.size() * 4, cudaMemcpyDeviceToHost));
    CKT(cudaMemcpy(bh.data(), bias, bh.size() * 4, cudaMemcpyDeviceToHost));
    rc = upload_conv_layer(h, L, wh, bh);
    if (rc) {
        cleanup();
        return rc;
    }
    const int Ho = (H + 2 * L.pad - k) / stride + 1, Wo = (W + 2 * L.pad - k) / stride + 1;
    Act in, out, r, p1, p2;
    in.N = B, in.H = H, in.W = W, in.C = Cin;
    out.N = B, out.H = Ho, out.W = Wo, out.C = L.Cout_pad;
    r = out;
    p1 = out;
    p2 = out;
    void* p = nullptr;
    CKT(cudaMalloc(&p, (size_t)in.plane() * 2 * h->planes));
    tmp.push_back(p);
    in.ptr = (__nv_bfloat16*)p;
    CKT(cudaMalloc(&p, (size_t)out.plane() * 2 * h->planes));
    tmp.push_back(p);
    out.ptr = (__nv_bfloat16*)p;
    CKT(cudaMemset(p, 0, (size_t)out.plane() * 2 * h->planes));  // TMA stores are invisible to initcheck
    CKT(launch_f32_to_split(x, in.ptr, in.plane(), in.plane(), h->planes, st, h->f16));
    const float* extra_src[3] = {res, post1, post2};
    Act* extra_act[3] = {&r, &p1, &p2};
    for (int e = 0; e < 3; e++) {
        if (!extra_src[e]) continue;
        if (L.Cout_pad != Cout) {
            cleanup();
            return fail(h, -1, "conv_test: residual/post operands require Cout % 32 == 0");
        }
        CKT(cudaMalloc(&p, (size_t)out.plane() * 2 * h->planes));
        tmp.push_back(p);
        extra_act[e]->ptr = (__nv_bfloat16*)p;
        CKT(launch_f32_to_split(extra_src[e], extra_act[e]->ptr, out.plane(), out.plane(), h->planes, st, h->f16));
    }
    ConvParams cp;
    int bn = 0;
    rc = setup_conv(h, L, in, res ? &r : nullptr, post1 ? &p1 : nullptr, post2 ? &p2 : nullptr, &out, nullptr, relu,
                    &cp, &bn, nullptr);
    if (rc) {
        cleanup();
        return rc;
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    long long* dbg_dev = nullptr;
    if (getenv("SMAPB_ROLES")) {
        CKT(cudaMalloc((void**)&dbg_dev, 16 * sizeof(long long)));
        tmp.push_back(dbg_dev);
        CKT(cudaMemset(dbg_dev, 0, 16 * sizeof(long long)));
        cp.dbg = dbg_dev;
    }
    long long* tl_dev = nullptr;
    if (getenv("SMAPB_TIMELINE")) {
        CKT(cudaMalloc((void**)&tl_dev, 16 * sizeof(long long)));
        tmp.push_back(tl_dev);
    }
    CKT(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st, false));  // warm-up + result
    if (dbg_dev) {
        long long d[16];
        CKT(cudaMemcpy(d, dbg_dev, sizeof d, cudaMemcpyDeviceToHost));
        const double n = d[ConvDbg::CTAS] > 0 ? (double)d[ConvDbg::CTAS] : 1.0;
        fprintf(stderr, "[roles] bn%d units%d kb%d | mean cycles per CTA: total %.0f | producer wait-empty %.0f", bn,
                cp.total_tiles, cp.kh * cp.kw * cp.kchunks + cp.kchunks2, d[ConvDbg::TOTAL] / n,
                d[ConvDbg::PRODUCER_WAIT_EMPTY] / n);
        for (int g = 0; g < 2; g++) {
            const long long* c = d + ConvDbg::CONS + ConvDbg::CONS_N * g;
            fprintf(stderr, " | g%d wait-full %.0f wait-order %.0f epilogue %.0f wait-ring %.0f wait-stage %.0f", g,
                    c[ConvDbg::WAIT_FULL] / n, c[ConvDbg::WAIT_ORDER] / n, c[ConvDbg::EPILOGUE] / n, c[ConvDbg::WAIT_RING] / n,
                    c[ConvDbg::WAIT_STAGE] / n);
        }
        fprintf(stderr, "\n");
        cp.dbg = nullptr;
    }
    if (tl_dev) {  // time line of CTA 0 of one warm launch (cycles since kernel entry)
        CKT(cudaMemset(tl_dev, 0, 16 * sizeof(long long)));
        cp.dbg_tl = tl_dev;
        CKT(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st, false));
        cp.dbg_tl = nullptr;
        long long t[16];
        CKT(cudaMemcpy(t, tl_dev, sizeof t, cudaMemcpyDeviceToHost));
        fprintf(stderr, "[timeline] bn%d units%d kb%d | set-up %lld | first operands %lld | last main loop end %lld | epilogue done "
                "%lld | exit %lld\n", bn, cp.total_tiles, cp.kh * cp.kw * cp.kchunks + cp.kchunks2, t[1] - t[0], t[2] - t[0],
                t[3] - t[0], t[13] - t[0], t[15] - t[0]);
    }
    const int reps = ms_out ? 5 : 0;
    cudaEventRecord(e0, st);
    for (int i = 0; i < reps; i++) CKT(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st, false));
    cudaEventRecord(e1, st);
    h->launches += 1 + reps;
    // de-pad + convert
    float* ytmp = nullptr;
    CKT(cudaMalloc((void**)&ytmp, (size_t)out.plane() * 4));
    tmp.push_back(ytmp);
    split_to_f32_kernel<<<(unsigned)((out.plane() + 255) / 256), 256, 0, st>>>(out.ptr, out.plane(), h->planes, ytmp,
                                                                               out.plane(), h->f16);
    CKT(cudaGetLastError());
    CKT(cudaMemcpy2DAsync(y, (size_t)Cout * 4, ytmp, (size_t)L.Cout_pad * 4, (size_t)Cout * 4, (size_t)B * Ho * Wo,
                          cudaMemcpyDeviceToDevice, st));
    CKT(cudaStreamSynchronize(st));
    if (ms_out) {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        *ms_out = ms / reps;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cleanup();
    return 0;
#undef CKT
}

#pragma GCC visibility pop
}  // extern "C"
