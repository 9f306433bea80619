// Internal to libsmap_b200 (not installed): the handle and plan types shared by engine.cu (handle, inference paths, C ABI)
// and plan.cu (conv set-up, tile choice, weights, execution plan).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdint.h>
#include <stdlib.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/smap_b200.h"
#include "conv_tc.cuh"
#include "decode_host.h"
#include "jpeg.h"
#include "jpeg_enc.h"
#include "png_enc.h"
#include "png.h"
#include "preprocess.h"
#include "refine.h"

namespace smapb {

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

struct ConvGeom {
    std::string name;
    int Cin = 0, Cout = 0, Cout_pad = 0, k = 1, stride = 1, pad = 0;
    int Cin2 = 0, stride2 = 1;  // K-concatenated second 1x1 input (weights hold Cin + Cin2 columns)
};
struct ConvLayer : ConvGeom {
    DeviceBuffer<__nv_bfloat16> w_dev;  // [T][taps][Cout_pad][Cin]
    DeviceBuffer<float> bias_dev;       // [Cout_pad]
};

enum OpKind { OP_STEM, OP_S2D, OP_MAXPOOL, OP_CONV, OP_HEADMERGE, OP_TAPSUM };
struct Op {
    OpKind kind;
    // conv
    ConvParams cp;
    int block_n = 0;
    double flops = 0;
    // generic tensors
    Act a, out;
    ActF32 f4, f3, f2;
    int cout = 0;  // head merge real channel count
    int which_out = 0;  // tap sum output: 1 detd, 2 rootd
    const float* bias = nullptr;  // tap-sum bias
    // two-stream execution: side-branch ops (skip convs, heads) run on stream 1 and overlap the main chain
    int stream = 0;
    std::vector<int> waits;  // indices of producer ops on the OTHER stream this op must wait for
    bool record = false;     // some op on the other stream consumes this op's output
    cudaEvent_t ev = nullptr;
    std::string name;  // reference unit name (NVTX range, profiles)
    // debug descriptions (smapb_debug_checksums): the tensors the op reads, in the order PlanBuilder::wire received them
    // (conv: ConvIO::inputs; null = role absent), and the output shape N, H, W, C of a conv
    std::vector<const void*> inputs;
    int dims[4] = {0, 0, 0, 0};
};

struct Plan {  // owns its tensors and the events of its ops
    Plan() = default;
    Plan(const Plan&) = delete;
    ~Plan() {
        for (Op& op : ops)
            if (op.ev) cudaEventDestroy(op.ev);
    }
    int B = 0;
    std::vector<Op> ops;
    std::vector<DeviceBuffer<uint8_t>> allocs;
    int n_conv = 0;
    double conv_flops = 0;
    std::map<const void*, int> producer;  // tensor -> index of the op that writes it (build time)
    int last_side = -1;
};

}  // namespace smapb

struct smapb_handle {
    int device = 0, max_batch = 0, in_h = 0, in_w = 0, h = 0, w = 0;
    int sm_count = 132;
    std::string err;
    int64_t launches = 0;
    // weights
    std::map<std::string, std::vector<float>> raw;
    std::map<std::string, std::vector<int64_t>> raw_shape;
    std::map<std::string, smapb::ConvLayer> layers;
    smapb::DeviceBuffer<float> stem_w;  // [147][64]
    smapb::ConvLayer stem_tc;  // space-to-depth tensor-core stem (4 ky-blocks x 64 k)
    int stem_tc_ok = -1;      // -1 untested, 0 overlapped TMA view rejected (CUDA-core stem), 1 in use
    smapb::DeviceBuffer<float> stem_b;
    int nterms = 3;  // MMA terms (3 = bf16x3, 1 = bf16 or fp16)
    int planes = 2;  // activation planes (2 or 1)
    bool f16 = false;  // element format of weights and activations: fp16 (SMAPB_PREC_FP16) instead of bf16
    smapb::DeviceBuffer<unsigned long long> sat_dev;  // fp16: activation elements clamped to +-65504 (smapb_saturation_count)
    bool finalized = false;
    std::map<int, std::unique_ptr<smapb::Plan>> plans;
    // association workspace (sized for max_batch)
    smapb::DeviceBuffer<float> peaks;
    smapb::DeviceBuffer<float> scores;
    smapb::DeviceBuffer<float> bodies;
    smapb::DeviceBuffer<int> counts;
    smapb::DeviceBuffer<uint32_t> nms_masks;  // one ballot bit per pixel of the key-point planes
    // whole-path workspace
    smapb::DeviceBuffer<float> imgs_dev;
    smapb::DeviceBuffer<float> imgs_flip;  // one allocation with hm_flip, scratch_detd and scratch_rootd
    smapb::DeviceBuffer<float> hm;
    float* hm_flip = nullptr;
    smapb::DeviceBuffer<float> detd;
    smapb::DeviceBuffer<float> rootd;
    float* scratch_detd = nullptr;
    float* scratch_rootd = nullptr;
    smapb::DeviceBuffer<double> scales_dev;
    smapb::DeviceBuffer<smapb_record> records_dev;
    // host-facing pipeline (smapb_submit_host / smapb_wait): two slots, H2D of slot s+1 overlaps the compute of slot s
    struct Slot {
        smapb::DeviceBuffer<float> imgs;
        smapb::DeviceBuffer<double> scales;
        smapb::DeviceBuffer<smapb_record> records;
        smapb::DeviceBuffer<smapb_record> records_all;  // [comm_world * max_batch], gathered variant
        cudaEvent_t h2d = nullptr, done = nullptr, rec_ready = nullptr;
        bool used = false;
    } slots[2];
    cudaStream_t copy_stream = nullptr;
    bool autotune = getenv("SMAPB_NO_AUTOTUNE") == nullptr;
    cudaStream_t aux_stream = nullptr;  // side branches of the decoder (skip convs, heads) run here
    // Stream used when the caller passes NULL (= the legacy default stream).  It is NON-blocking - a blocking stream would
    // be fenced by every legacy-stream operation of the process (e.g. a collective issued by the host framework) - and is
    // ordered against the legacy stream explicitly with the two bridge events (on_stream in engine.cu).
    cudaStream_t own_stream = nullptr;
    cudaEvent_t bridge_in = nullptr, bridge_out = nullptr;
    struct GraphEntry {
        int B, flip, gather;
        const void* imgs;
        const void* scales;
        cudaGraphExec_t exec;
        uint64_t stamp;  // last use (LRU eviction)
        int64_t launches;  // counted while the graph was captured; each replay adds them to `launches`
    };
    std::vector<GraphEntry> graphs;  // whole-path CUDA graphs keyed by (B, flip, gather, input pointers)
    uint64_t graph_clock = 0;
    // skeleton-record exchange (SURVEY 8(e)): one ncclAllGather per batch on the compute stream, inside the graph
    void* comm = nullptr;  // ncclComm_t
    bool comm_owned = false;
    int comm_rank = 0, comm_world = 1;
    smapb::DeviceBuffer<smapb_record> gather_dev;  // [comm_world * max_batch]
    // decoupled exchange (smapb_infer_device_gather_async / smapb_submit_host_gather): the all-gather runs on its own stream
    // behind an event, so a rank's compute stream never waits for its peers
    cudaStream_t gather_stream = nullptr;
    cudaEvent_t rec_ready[2] = {nullptr, nullptr}, gather_done[2] = {nullptr, nullptr};
    smapb::DeviceBuffer<smapb_record> rec_buf;  // [2][max_batch]: the two latest async calls' records
    bool gather_used[2] = {false, false};
    int gather_idx = 0;
    smapb::DeviceBuffer<double> gt_dist;  // [max_batch][127*127] distance matrices of the GT-matching lift
    bool nccl_in_graph = getenv("SMAPB_NCCL_EAGER") == nullptr;
    bool nvtx_ops = getenv("SMAPB_NVTX") != nullptr;  // one NVTX range per plan op (phase ranges are always emitted)
    // pre-processing (SURVEY 8(f) f1): resampling tables per source geometry, staging for host images
    struct PreEntry {
        smapb::ResizePlan plan;
        smapb::ResizeTablesDev tab{};
        smapb::DeviceBuffer<char> buf;
    };
    std::map<std::pair<int, int>, PreEntry> pre_cache;
    smapb::DeviceBuffer<uint8_t> pre_stage;
    // JPEG decoding (smapb_decode_jpeg), PNG decoding (smapb_decode_png), JPEG encoding (smapb_encode_jpeg) and PNG
    // encoding (smapb_encode_png), created on first use
    std::unique_ptr<smapb::JpegWorkspace, void (*)(smapb::JpegWorkspace*)> jpeg{nullptr, smapb::jpeg_workspace_destroy};
    std::unique_ptr<smapb::PngWorkspace, void (*)(smapb::PngWorkspace*)> png{nullptr, smapb::png_workspace_destroy};
    std::unique_ptr<smapb::JpegEncWorkspace, void (*)(smapb::JpegEncWorkspace*)> jpeg_enc{nullptr,
                                                                                          smapb::jpeg_enc_workspace_destroy};
    std::unique_ptr<smapb::PngEncWorkspace, void (*)(smapb::PngEncWorkspace*)> png_enc{nullptr, smapb::png_enc_workspace_destroy};
    // RefineNet (optional post-processing step, SURVEY 8(f) f2)
    std::map<std::string, std::vector<float>> refine_raw;
    smapb::DeviceBuffer<float> refine_buf;  // folded, transposed weights + biases of the five layers
    smapb::RefineWeights refine_w{};
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
    smapb::DeviceBuffer<long long> roles_dev;  // [ROLES_CAP][16]
    size_t roles_used = 0;
    std::vector<std::string> roles_desc;
};

namespace smapb {

constexpr size_t ROLES_CAP = 4096;

inline int fail(smapb_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    return code;
}
#define CK(call)                                                                                          \
    do {                                                                                                  \
        cudaError_t e_ = (call);                                                                          \
        if (e_ != cudaSuccess)                                                                            \
            return fail(h, -10, std::string(#call) + ": " + cudaGetErrorString(e_) + " @" + std::to_string(__LINE__)); \
    } while (0)

template <typename T>
int dev_alloc(smapb_handle* h, DeviceBuffer<T>& b, size_t count) {  // b.grow(count), its failure reported as fail() does
    const cudaError_t e = b.grow(count);
    return e == cudaSuccess ? 0 : fail(h, -10, std::string("cudaMalloc: ") + cudaGetErrorString(e));
}

struct NvtxScope {  // NVTX range that every return from its scope pops; next() ends it and opens the next one
    const bool on;
    explicit NvtxScope(const char* name, bool enable = true) : on(enable) { if (on) nvtxRangePushA(name); }
    void next(const char* name) { if (on) nvtxRangePop(), nvtxRangePushA(name); }
    ~NvtxScope() { if (on) nvtxRangePop(); }
};

enum ProfKind { PK_START = -1, PK_CONV = 0, PK_STEM = 1, PK_ELEM = 2, PK_ASSOC = 3, PK_LIFT = 4, PK_COPY = 5 };
inline void prof_mark(smapb_handle* h, int kind, cudaStream_t st, const char* desc = "", double flops = 0) {
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

// plan.cu
int build_plan(smapb_handle* h, int B, Plan** out_plan);
int run_plan(smapb_handle* h, Plan* plan, const float* imgs, float* hm2d, float* detd, float* rootd, cudaStream_t st);
// engine.cu
void drop_graphs(smapb_handle* h, bool gather_only = false);  // destroys the cached whole-path graphs (or those with the all-gather)

}  // namespace smapb
