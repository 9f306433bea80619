// Host side of libsmap_b200: handle life cycle, the inference, graph and gather paths, NCCL, pre-processing, JPEG, RefineNet
// and profiling entry points of the C ABI (include/smap_b200.h).  The execution plan and the weights are in plan.cu.
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "../../include/smap_b200_debug.h"
#include "assoc.h"
#include "elementwise.h"
#include "engine.h"

using namespace smapb;

namespace {

thread_local std::string g_create_error = "";

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

// Runs body(stream) on the caller's stream or, for NULL (the legacy default stream, which cannot be captured into a graph),
// on the handle's own non-blocking stream: ordered after the legacy stream's pending work and, once the body succeeded, the
// legacy stream after it - what a blocking stream would give the caller, without fencing every other stream of the process.
template <class F>
int on_stream(smapb_handle* h, void* stream, F&& body) {
    if (stream) return body((cudaStream_t)stream);
    CK(cudaEventRecord(h->bridge_in, cudaStreamLegacy));
    CK(cudaStreamWaitEvent(h->own_stream, h->bridge_in, 0));
    const int rc = body(h->own_stream);
    if (rc) return rc;
    CK(cudaEventRecord(h->bridge_out, h->own_stream));
    CK(cudaStreamWaitEvent(cudaStreamLegacy, h->bridge_out, 0));
    return 0;
}

// Every stream and every event of a handle.  smapb_create makes them all, so that the lazy set-ups of the whole path only
// allocate device memory; smapb_destroy destroys those that exist.
std::vector<cudaStream_t*> handle_streams(smapb_handle* h) {
    return {&h->own_stream, &h->aux_stream, &h->copy_stream, &h->gather_stream};
}
std::vector<cudaEvent_t*> handle_events(smapb_handle* h) {
    return {&h->bridge_in, &h->bridge_out, &h->rec_ready[0], &h->rec_ready[1], &h->gather_done[0], &h->gather_done[1],
            &h->slots[0].h2d, &h->slots[0].done, &h->slots[0].rec_ready, &h->slots[1].h2d, &h->slots[1].done,
            &h->slots[1].rec_ready};
}

}  // namespace

void smapb::drop_graphs(smapb_handle* h, bool gather_only) {
    auto dropped = [&](const smapb_handle::GraphEntry& g) { return !gather_only || g.gather; };
    for (auto& g : h->graphs)
        if (dropped(g)) cudaGraphExecDestroy(g.exec);
    h->graphs.erase(std::remove_if(h->graphs.begin(), h->graphs.end(), dropped), h->graphs.end());
}

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
    const size_t hw = (size_t)h->h * h->w;
    const size_t MB = max_batch;
    int rc = 0;
    rc |= dev_alloc(h, h->peaks, MB * NJ * (MAXP + 1) * 3);
    rc |= dev_alloc(h, h->scores, MB * NL * MAXP * MAXP);
    rc |= dev_alloc(h, h->bodies, MB * MAXP * NJ * 4);
    rc |= dev_alloc(h, h->counts, MB);
    rc |= dev_alloc(h, h->nms_masks, nms_mask_words(max_batch, h->h, h->w));
    rc |= dev_alloc(h, h->imgs_dev, MB * 3 * in_h * in_w);
    rc |= dev_alloc(h, h->hm, MB * NC2D * hw);
    rc |= dev_alloc(h, h->detd, MB * NL * hw);
    rc |= dev_alloc(h, h->rootd, MB * hw);
    rc |= dev_alloc(h, h->scales_dev, MB * SMAPB_SCALE_LEN);
    rc |= dev_alloc(h, h->records_dev, MB);
    rc |= dev_alloc(h, h->sat_dev, 1);
    if (!rc && cudaMemset(h->sat_dev, 0, sizeof(unsigned long long)) != cudaSuccess) rc = -10;
    if (rc) {
        g_create_error = h->err;
        delete h;
        return -10;
    }
    bool made = true;
    for (cudaStream_t* s : handle_streams(h)) made = made && cudaStreamCreateWithFlags(s, cudaStreamNonBlocking) == cudaSuccess;
    for (cudaEvent_t* e : handle_events(h)) made = made && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
    if (!made) {
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
    drop_graphs(h);
    if (h->comm && h->comm_owned && nccl_api().CommDestroy) nccl_api().CommDestroy(h->comm);
    for (cudaStream_t* s : handle_streams(h))
        if (*s) cudaStreamDestroy(*s);
    for (cudaEvent_t* e : handle_events(h))
        if (*e) cudaEventDestroy(*e);
    for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
    delete h;  // the plans, weights, buffers and codec workspaces free themselves
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

int smapb_backbone_forward(smapb_handle* h, const float* imgs, int B, float* hm2d, float* detd, float* rootd,
                           void* stream) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, "smapb_backbone_forward: weights not finalized");
    if (B < 1) return fail(h, -1, "B < 1");
    cudaSetDevice(h->device);
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
    if (rc) return rc;
    return on_stream(h, stream, [&](cudaStream_t st) { return run_plan(h, plan, imgs, hm2d, detd, rootd, st); });
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
    if (dev_alloc(h, h->gt_dist, (size_t)h->max_batch * MAXP * MAXP)) return -10;
    CK(launch_lift_gt(bodies, counts, detd, rootd, scales, gt_roots, gt_counts, gmax, h->gt_dist, B, h->h, h->w, 2, pred2d,
                      pred3d, root_depth, counts_out, (cudaStream_t)stream));
    h->launches++;
    return 0;
}

// ---- pre-processing (SURVEY 8(f) f1) ---------------------------------------------------------------------------
static int pre_entry(smapb_handle* h, int img_h, int img_w, smapb_handle::PreEntry** out) {
    auto key = std::make_pair(img_w, img_h);
    auto it = h->pre_cache.find(key);
    if (it == h->pre_cache.end()) {
        smapb_handle::PreEntry E;
        if (!make_resize_plan(img_w, img_h, h->in_w, h->in_h, &E.plan)) {
            char msg[256];
            snprintf(msg, sizeof msg,
                     "smapb_preprocess: a %dx%d image (W x H) does not fit a %dx%d input: sides must be in [1, 16384] and "
                     "resize to at least 1 pixel (cv2.resize refuses an empty size)",
                     img_w, img_h, h->in_w, h->in_h);
            return fail(h, -1, msg);
        }
        if (h->pre_cache.size() >= 256) {  // bound the cache: drop everything (streams are idle after the sync)
            cudaDeviceSynchronize();
            h->pre_cache.clear();
        }
        const ResizePlan& P = E.plan;
        const size_t nx = P.xofs.size(), ny = P.yofs.size();  // ny = 2 * dst_h
        const size_t bytes = nx * 4 + ny * 4 + nx * 2 * 2 + ny * 2 + 64;
        CK(E.buf.grow(bytes));
        int* xo = (int*)E.buf.get();
        int* yo = xo + nx;
        short* xc = (short*)(yo + ny);
        short* yc = xc + 2 * nx;
        cudaError_t ce = cudaMemcpy(xo, P.xofs.data(), nx * 4, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(yo, P.yofs.data(), ny * 4, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(xc, P.xcoef.data(), nx * 2 * 2, cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(yc, P.ycoef.data(), ny * 2, cudaMemcpyHostToDevice);
        if (ce != cudaSuccess) return fail(h, -10, std::string("smapb_preprocess: table upload: ") + cudaGetErrorString(ce));
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
    smapb_handle::PreEntry* E = nullptr;
    int rc = pre_entry(h, img_h, img_w, &E);  // refuse the geometry before staging its pixels
    if (rc) return rc;
    const size_t bytes = (size_t)img_h * img_w * 3;
    if (bytes > h->pre_stage.capacity()) {
        cudaDeviceSynchronize();  // a pending copy may still read the old staging buffer
        CK(h->pre_stage.grow(bytes));
    }
    CK(cudaMemcpyAsync(h->pre_stage, bgr_host, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return smapb_preprocess(h, h->pre_stage, img_h, img_w, out_nchw_dev, scale_row_host, stream);
}

int smapb_decode_jpeg_ex(smapb_handle* h, int n, const uint8_t* const* jpeg_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                         int flags, int* status_host, void* stream) {
    if (!h) return -1;
    if (flags & ~(SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR)) {
        h->err = "smapb_decode_jpeg_ex: unknown flags";
        return -1;
    }
    cudaSetDevice(h->device);
    if (!h->jpeg) h->jpeg.reset(smapb::jpeg_workspace_create());
    return smapb::jpeg_decode(h->jpeg.get(), n, jpeg_host, nbytes, bgr_dev, flags, status_host, (cudaStream_t)stream, &h->launches,
                              &h->err);
}

int smapb_decode_jpeg(smapb_handle* h, int n, const uint8_t* const* jpeg_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                      int* status_host, void* stream) {
    return smapb_decode_jpeg_ex(h, n, jpeg_host, nbytes, bgr_dev, 0, status_host, stream);
}

int smapb_decode_png(smapb_handle* h, int n, const uint8_t* const* png_host, const int64_t* nbytes, uint8_t* const* bgr_dev,
                     int* status_host, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    if (!h->png) h->png.reset(smapb::png_workspace_create());
    return smapb::png_decode(h->png.get(), n, png_host, nbytes, bgr_dev, status_host, (cudaStream_t)stream, &h->launches, &h->err);
}

int smapb_encode_jpeg_ex(smapb_handle* h, int n, const uint8_t* const* bgr_dev, const int* img_h, const int* img_w, int quality,
                         const smapb_record* records_dev, const double* scales_dev, int flags, int64_t* nbytes_host, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    if (!h->jpeg_enc) h->jpeg_enc.reset(smapb::jpeg_enc_workspace_create());
    return smapb::jpeg_encode(h->jpeg_enc.get(), n, bgr_dev, img_h, img_w, quality, records_dev, scales_dev, flags, nbytes_host,
                              (cudaStream_t)stream, &h->launches, &h->err);
}

int smapb_encode_jpeg(smapb_handle* h, int n, const uint8_t* const* bgr_dev, const int* img_h, const int* img_w, int quality,
                      const smapb_record* records_dev, const double* scales_dev, int64_t* nbytes_host, void* stream) {
    return smapb_encode_jpeg_ex(h, n, bgr_dev, img_h, img_w, quality, records_dev, scales_dev, 0, nbytes_host, stream);
}

int smapb_encoded_jpeg(const smapb_handle* h, int i, const uint8_t** data, int64_t* nbytes) {
    if (!h || !data) return -1;
    *data = smapb::jpeg_enc_result(h->jpeg_enc.get(), i, nbytes);
    return *data ? 0 : -1;
}

int smapb_png_inflate_stats(const smapb_handle* h, int64_t* counts4) {
    if (!h || !counts4) return -1;
    smapb::png_last_stats(h->png.get(), counts4);
    return 0;
}

// host-only introspection of the resampling plan (tests compare it with the oracle over many geometries without a GPU)
int smapb_debug_resize_plan(int src_w, int src_h, int net_w, int net_h, int* dims6, double* scale, int* xofs, short* xcoef,
                            int* yofs, short* ycoef) {
    ResizePlan P;
    if (!dims6 || !make_resize_plan(src_w, src_h, net_w, net_h, &P)) return -1;
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
    CK(h->refine_buf.grow(total));
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
        drop_graphs(h);
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

// A smapb_record array as the lift and RefineNet kernels take it: record 0's fields, and the record stride in 4 and 8 bytes
struct RecordFields {
    float* pred2d;
    double *pred3d, *root_depth;
    int* count;
    static constexpr long long s4 = sizeof(smapb_record) / 4, s8 = sizeof(smapb_record) / 8;
    explicit RecordFields(smapb_record* r)
        : pred2d(r->pred2d[0][0]), pred3d(r->pred3d[0][0]), root_depth(r->root_depth), count(&r->count) {}
};

static int infer_body(smapb_handle* h, Plan* plan, const float* imgs, const double* scales, int B, int do_flip,
                      smapb_record* records, cudaStream_t st) {
    NvtxScope range("smapb.backbone");
    if (int rc = run_plan(h, plan, imgs, h->hm, h->detd, h->rootd, st)) return rc;
    if (do_flip) {
        if (!h->imgs_flip) {  // one allocation, so that a failed set-up leaves nothing behind and is tried again
            const size_t MB = h->max_batch, hw = (size_t)h->h * h->w, frames = MB * 3 * h->in_h * h->in_w;
            if (dev_alloc(h, h->imgs_flip, frames + MB * (NC2D + NL + 1) * hw)) return -10;
            h->hm_flip = h->imgs_flip + frames;  // every part 256-byte aligned: in_h and in_w are multiples of 32
            h->scratch_detd = h->hm_flip + MB * NC2D * hw;
            h->scratch_rootd = h->scratch_detd + MB * NL * hw;
        }
        flip_w_kernel<<<132 * 8, 256, 0, st>>>(imgs, h->imgs_flip, (long long)B * 3 * h->in_h, h->in_w);
        CK(cudaGetLastError());
        prof_mark(h, PK_ELEM, st, "flip_w");
        h->launches++;
        if (int rc = run_plan(h, plan, h->imgs_flip, h->hm_flip, h->scratch_detd, h->scratch_rootd, st)) return rc;
    }
    range.next("smapb.association");
    CK(launch_merge_scale(h->hm, do_flip ? h->hm_flip : nullptr, B, h->h, h->w, 1, st));
    prof_mark(h, PK_ELEM, st, "merge_scale");
    CK(launch_nms(h->hm, NC2D, B, h->h, h->w, 0.2f, h->peaks, h->nms_masks, st));
    prof_mark(h, PK_ASSOC, st, "nms");
    CK(launch_paf(h->hm, NC2D, B, h->h, h->w, h->peaks, h->scores, 0, st));
    prof_mark(h, PK_ASSOC, st, "paf");
    CK(launch_group(h->peaks, h->scores, h->rootd, B, h->h, h->w, 2, 1, h->bodies, h->counts, st));
    prof_mark(h, PK_ASSOC, st, "group");
    range.next("smapb.lift");
    const RecordFields r(records);
    CK(launch_lift(h->bodies, h->counts, h->detd, h->rootd, scales, B, h->h, h->w, 2, r.pred2d, r.pred3d, r.root_depth,
                   r.count, r.s4, r.s8, r.s8, r.s4, st));
    prof_mark(h, PK_LIFT, st, "lift");
    h->launches += 6;
    if (h->refine_on) {  // refined poses replace pred3d, as save_result(pred_bodys_2d, new_pred_bodys_3d, ...) does (test.py:137-145)
        CK(launch_refine_records(h->refine_w, r.pred2d, r.pred3d, r.count, B, 2, r.s4, r.s8, r.s4, r.pred3d, r.s8, st));
        prof_mark(h, PK_LIFT, st, "refine");
        h->launches++;
    }
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

// What every whole-path entry needs, checked before the entry changes any state of the handle; selects the handle's device.
// gather: the records are exchanged over the handle's communicator.  slot: that of the submit forms, 0 for the others.
static int check_whole_path(smapb_handle* h, const char* fn, int B, bool gather, int slot = 0) {
    if (!h) return -1;
    if (!h->finalized) return fail(h, -2, std::string(fn) + ": weights not finalized");
    if (slot < 0 || slot > 1) return fail(h, -1, std::string(fn) + ": slot must be 0 or 1");
    if (gather && (!h->comm || !h->gather_dev))  // gather_dev: allocated when the communicator was attached
        return fail(h, -52, std::string(fn) + ": no communicator attached (smapb_comm_create / smapb_comm_attach)");
    cudaSetDevice(h->device);
    return check_assoc(h, B);  // B in [1, max_batch], and a map size the association can stage
}

// Whole path on stream `st` (never NULL here), for arguments check_whole_path accepted.  gather != 0: followed by the
// all-gather of the records over the handle's communicator; `records` then receives comm_world * B records in rank order.
static int infer_device_impl(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip, int gather,
                             smapb_record* records, cudaStream_t st) {
    Plan* plan = nullptr;
    int rc = build_plan(h, B, &plan);
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
        const int64_t launches = h->launches - launches_before;
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
        h->graphs.push_back({B, do_flip, gather, imgs, scales, exec, 0, launches});
        ge = &h->graphs.back();
    }
    ge->stamp = ++h->graph_clock;
    CK(cudaGraphLaunch(ge->exec, st));
    h->launches += ge->launches;
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

// The exchange behind an event: the gather stream waits until `st` has written `send`, all-gathers it into `recv` and,
// with `host`, copies the comm_world * B records there; `done` marks the end of it on the gather stream.
static int decoupled_exchange(smapb_handle* h, cudaStream_t st, const smapb_record* send, smapb_record* recv, int B,
                              smapb_record* host, cudaEvent_t ready, cudaEvent_t done) {
    CK(cudaEventRecord(ready, st));
    CK(cudaStreamWaitEvent(h->gather_stream, ready, 0));
    if (int rc = gather_records(h, h->comm, send, recv, B, h->gather_stream)) return rc;
    if (host)
        CK(cudaMemcpyAsync(host, recv, (size_t)B * h->comm_world * sizeof(smapb_record), cudaMemcpyDeviceToHost,
                           h->gather_stream));
    CK(cudaEventRecord(done, h->gather_stream));
    return 0;
}

static int infer_device_entry(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip, int gather,
                              smapb_record* records, void* stream) {
    if (int rc = check_whole_path(h, gather ? "smapb_infer_device_gather" : "smapb_infer_device", B, gather)) return rc;
    return on_stream(h, stream,
                     [&](cudaStream_t st) { return infer_device_impl(h, imgs, scales, B, do_flip, gather, records, st); });
}

int smapb_infer_device(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                       smapb_record* records, void* stream) {
    return infer_device_entry(h, imgs, scales, B, do_flip, 0, records, stream);
}

int smapb_infer_device_gather(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                              smapb_record* all_records, void* stream) {
    return infer_device_entry(h, imgs, scales, B, do_flip, 1, all_records, stream);
}

// Whole path on the caller's stream, exchange on the handle's gather stream: the caller's stream is ordered after the COMPUTE
// only.  all_records is valid once smapb_gather_sync has made a stream wait for the exchange.  The records are
// double-buffered, so a call only waits for the exchange issued two calls earlier.
int smapb_infer_device_gather_async(smapb_handle* h, const float* imgs, const double* scales, int B, int do_flip,
                                    smapb_record* all_records, void* stream) {
    if (int rc = check_whole_path(h, "smapb_infer_device_gather_async", B, true)) return rc;
    // both in one allocation, so that a failed set-up leaves nothing behind and is tried again
    if (dev_alloc(h, h->rec_buf, 2 * (size_t)h->max_batch)) return -10;
    return on_stream(h, stream, [&](cudaStream_t st) {
        const int idx = h->gather_idx;
        h->gather_idx ^= 1;
        if (h->gather_used[idx]) CK(cudaStreamWaitEvent(st, h->gather_done[idx], 0));
        smapb_record* const rec = h->rec_buf + (size_t)idx * h->max_batch;
        int rc = infer_device_impl(h, imgs, scales, B, do_flip, 0, rec, st);
        if (!rc) rc = decoupled_exchange(h, st, rec, all_records, B, nullptr, h->rec_ready[idx], h->gather_done[idx]);
        if (rc) return rc;
        h->gather_used[idx] = true;
        return 0;
    });
}

int smapb_gather_sync(smapb_handle* h, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    cudaStream_t st = stream ? (cudaStream_t)stream : cudaStreamLegacy;
    for (int i = 0; i < 2; i++)
        if (h->gather_used[i]) CK(cudaStreamWaitEvent(st, h->gather_done[i], 0));
    return 0;
}

static int upload_batch(smapb_handle* h, const float* imgs, const double* scales, int B, float* to_imgs, double* to_scales,
                        cudaStream_t st) {  // the B frames and scale rows of a host batch
    CK(cudaMemcpyAsync(to_imgs, imgs, (size_t)B * 3 * h->in_h * h->in_w * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(to_scales, scales, (size_t)B * SMAPB_SCALE_LEN * sizeof(double), cudaMemcpyHostToDevice, st));
    return 0;
}

int smapb_infer_host(smapb_handle* h, const float* imgs_host, const double* scales_host, int B, int do_flip,
                     smapb_record* records_host, void* stream) {
    if (int rc = check_whole_path(h, "smapb_infer_host", B, false)) return rc;
    return on_stream(h, stream, [&](cudaStream_t st) {
        int rc = upload_batch(h, imgs_host, scales_host, B, h->imgs_dev, h->scales_dev, st);
        if (!rc) rc = infer_device_impl(h, h->imgs_dev, h->scales_dev, B, do_flip, 0, h->records_dev, st);
        if (rc) return rc;
        CK(cudaMemcpyAsync(records_host, h->records_dev, (size_t)B * sizeof(smapb_record), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    });
}

static int submit_host_impl(smapb_handle* h, int slot, const float* imgs_host, const double* scales_host, int B, int do_flip,
                            int gather, smapb_record* records_host) {
    if (int rc = check_whole_path(h, gather ? "smapb_submit_host_gather" : "smapb_submit_host", B, gather, slot)) return rc;
    smapb_handle::Slot& S = h->slots[slot];
    if (!S.imgs) {  // into locals first, so that a failed set-up leaves nothing behind and is tried again
        const size_t MB = h->max_batch;
        DeviceBuffer<float> imgs;
        DeviceBuffer<double> scales;
        DeviceBuffer<smapb_record> records;
        if (dev_alloc(h, imgs, MB * 3 * h->in_h * h->in_w) || dev_alloc(h, scales, MB * SMAPB_SCALE_LEN) ||
            dev_alloc(h, records, MB))
            return -10;
        S.imgs = std::move(imgs), S.scales = std::move(scales), S.records = std::move(records);
    }
    if (gather && dev_alloc(h, S.records_all, (size_t)h->max_batch * h->comm_world)) return -10;
    // the slot's buffers are free once its previous submission has completed
    if (S.used) CK(cudaStreamWaitEvent(h->copy_stream, S.done, 0));
    if (int rc = upload_batch(h, imgs_host, scales_host, B, S.imgs, S.scales, h->copy_stream)) return rc;
    CK(cudaEventRecord(S.h2d, h->copy_stream));
    cudaStream_t st = h->own_stream;
    CK(cudaStreamWaitEvent(st, S.h2d, 0));
    if (int rc = infer_device_impl(h, S.imgs, S.scales, B, do_flip, 0, S.records, st)) return rc;
    if (!gather) {
        CK(cudaMemcpyAsync(records_host, S.records, (size_t)B * sizeof(smapb_record), cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(S.done, st));
    } else {
        // The exchange and the D2H of its result run on the gather stream: the compute stream goes straight on to the next
        // slot's batch and never waits for a peer.  The records are exchanged on the device (NVLink) and leave in ONE D2H -
        // nothing is re-uploaded.
        if (int rc = decoupled_exchange(h, st, S.records, S.records_all, B, records_host, S.rec_ready, S.done)) return rc;
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
    drop_graphs(h, true);
    for (auto& kv : h->eager_runs)
        if (kv.first.second & 1) kv.second = 0;
    h->comm = comm, h->comm_owned = owned, h->comm_rank = rank, h->comm_world = world;
    h->gather_dev.reset();
    for (auto& S : h->slots) S.records_all.reset();
    if (dev_alloc(h, h->gather_dev, (size_t)world * h->max_batch)) return -10;
    return 0;
}

int smapb_comm_create(smapb_handle* h, const void* id128, int rank, int world) {
    if (!h || !id128) return -1;
    NcclApi& a = nccl_api();
    if (!a.lib) return fail(h, -51, a.err.empty() ? "NCCL unavailable" : a.err);
    // refused here, before NCCL sees them: ncclCommInitRank would otherwise be the one to judge rank and world
    if (world < 1 || rank < 0 || rank >= world) return fail(h, -1, "communicator: rank / world out of range");
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
    return on_stream(h, stream, [&](cudaStream_t st) { return gather_records(h, comm, records_dev, all_records_dev, B, st); });
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
        CK(h->roles_dev.grow(ROLES_CAP * 16));
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

#pragma GCC visibility pop
}  // extern "C"
