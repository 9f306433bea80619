// Execution plan of libsmap_b200's backbone: conv set-up and tile choice, BN folding and weight repacking, the plan builder,
// the plan runner, and the C ABI entry points that work on them (include/smap_b200.h, include/smap_b200_debug.h).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "../../include/smap_b200_debug.h"
#include "elementwise.h"
#include "engine.h"

using namespace smapb;

namespace {

// Process-wide tile-shape table: layer geometry -> (BLOCK_N, CTAs per tile).  Filled from the committed table
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

// The tensors of one conv.  `in` is required, the others are optional (null = absent): in2 is the K-concatenated second
// input of a fused pair, res a residual added before the ReLU, post1 / post2 tensors added after it, up the low-resolution
// tensor of the fused bilinear x2 residual.  The conv writes `out` (split planes) or `out_f32`.
struct ConvIO {
    const Act* in = nullptr;
    int relu = 0;
    const Act *in2 = nullptr, *res = nullptr, *post1 = nullptr, *post2 = nullptr, *up = nullptr, *out = nullptr;
    const ActF32* out_f32 = nullptr;
    // the tensors the conv reads, in the role order of CONV_ROLES
    std::vector<const void*> inputs() const {
        auto p = [](const Act* a) -> const void* { return a ? a->ptr : nullptr; };
        return {in->ptr, p(res), p(post1), p(post2), p(in2), p(up)};
    }
};
const char* const CONV_ROLES[6] = {"in", "res", "p1", "p2", "in2", "up"};

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
cudaError_t launch_conv_inst2(const ConvParams& cp, int sm_count, cudaStream_t st) {
    using Cfg = ConvCfg<BN, NT, RING>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, NT, RING, E>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    const int units = cp.total_tiles < sm_count ? cp.total_tiles : sm_count;  // persistent CTAs
    conv_tc_kernel<BN, NT, RING, E><<<units, 384, Cfg::SMEM_BYTES, st>>>(cp);
    return cudaGetLastError();
}
// The RING variant a conv runs: 2 = fused bilinear residual, 1 = residual / skip tensors, 0 = no epilogue inputs
int conv_ring(const ConvParams& cp) { return cp.up_mode ? 2 : (cp.has_res + cp.n_post) ? 1 : 0; }
template <int BN, int NT, class E = ElemBF16>
cudaError_t launch_conv_inst(const ConvParams& cp, int sm_count, cudaStream_t st) {
    switch (conv_ring(cp)) {
        case 2: return launch_conv_inst2<BN, NT, 2, E>(cp, sm_count, st);
        case 1: return launch_conv_inst2<BN, NT, 1, E>(cp, sm_count, st);
        default: return launch_conv_inst2<BN, NT, 0, E>(cp, sm_count, st);
    }
}
cudaError_t launch_conv(const ConvParams& cp, int block_n, int nterms, bool f16, int sm_count, cudaStream_t st) {
#define SMAPB_CASE(BN)                                                             \
    case BN:                                                                       \
        if (f16) return launch_conv_inst<BN, 1, ElemF16>(cp, sm_count, st);        \
        return nterms == 3 ? launch_conv_inst<BN, 3>(cp, sm_count, st)             \
                           : launch_conv_inst<BN, 1>(cp, sm_count, st);
    switch (block_n) {
        SMAPB_CASE(128)
        SMAPB_CASE(64)
        SMAPB_CASE(32)
    }
#undef SMAPB_CASE
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------
// conv set-up
// ------------------------------------------------------------------------------------------------
// The tile widths the kernel is built for: one CTA per tile of 128 output pixels x 32, 64 or 128 channels
bool tile_shape_ok(int bn) { return bn == 32 || bn == 64 || bn == 128; }

// The tw x (128 / tw) output patch with the fewest wasted pixels.  smax: the largest input stride (an input box spans at most
// 256 pixels); up: the low-resolution patch of a fused bilinear residual must fit one ring slot.
int patch_width(int Ho, int Wo, int smax, bool up) {
    double best = -1;
    int tw = 16;
    for (int c = 128; c >= 1; c >>= 1) {
        const int t_h = 128 / c;
        if (c * smax > 256 || t_h * smax > 256) continue;
        if (up && (c / 2 + 2) * (t_h / 2 + 2) > 128) continue;
        const double util = ((double)Wo * Ho) / ((double)((Wo + c - 1) / c) * c * ((Ho + t_h - 1) / t_h) * t_h);
        if (util > best + 1e-9) {
            best = util;
            tw = c;
        }
    }
    return tw;
}

// The tiling fields of *cp: nimg images of Hout x Wout output pixels in patches of tw x (128 / tw), n_tiles channel tiles
void set_tiling(ConvParams* cp, int nimg, int Hout, int Wout, int tw, int n_tiles) {
    const int th = 128 / tw;
    int twl = 0;
    while ((1 << twl) < tw) twl++;
    cp->Nimg = nimg;
    cp->Hout = Hout;
    cp->Wout = Wout;
    cp->tw_log2 = twl;
    cp->th = th;
    cp->tiles_x = (Wout + tw - 1) / tw;
    cp->tiles_y = (Hout + th - 1) / th;
    cp->n_tiles = n_tiles;
    cp->total_tiles = (int)((long long)cp->tiles_x * cp->tiles_y * nimg * n_tiles);
}

// Flat convs (1x1, stride 1, no up-residual) see their N x Ho x Wo output pixels as one row of 128-pixel tiles
bool is_flat(const ConvLayer& L, const ConvIO& io) {
    return L.k == 1 && L.stride == 1 && (!io.in2 || L.stride2 == 1) && !io.up;
}
void conv_tiling(const ConvLayer& L, const ConvIO& io, int n_tiles, ConvParams* cp) {
    const Act& in = *io.in;
    const int Ho = (in.H + 2 * L.pad - L.k) / L.stride + 1, Wo = (in.W + 2 * L.pad - L.k) / L.stride + 1;
    if (is_flat(L, io))
        set_tiling(cp, 1, 1, (int)((long long)in.N * Ho * Wo), 128, n_tiles);
    else
        set_tiling(cp, in.N, Ho, Wo, patch_width(Ho, Wo, io.in2 ? std::max(L.stride, L.stride2) : L.stride, io.up),
                   n_tiles);
}

// Fill a ConvParams for `L` applied to io's tensors, with tiles of block_n output channels.
int setup_conv(smapb_handle* h, const ConvLayer& L, const ConvIO& io, int block_n, ConvParams* cp) {
    const Act& in = *io.in;
    const Act *in2 = io.in2, *res = io.res, *post1 = io.post1, *post2 = io.post2, *up = io.up;
    if (in.C != L.Cin) return fail(h, -30, "conv " + L.name + ": Cin mismatch");
    if (L.Cin % 64 != 0) return fail(h, -30, "conv " + L.name + ": Cin must be a multiple of 64");
    memset(cp, 0, sizeof(*cp));
    if ((L.Cin2 != 0) != (in2 != nullptr)) return fail(h, -30, "conv " + L.name + ": second input mismatch");
    if (L.Cin2 % 64 != 0) return fail(h, -30, "conv " + L.name + ": Cin2 must be a multiple of 64");
    if (in2 && (in2->C != L.Cin2 || L.k != 1 || L.stride != 1)) return fail(h, -30, "conv " + L.name + ": bad fused pair");
    if (up && (res || post1)) return fail(h, -30, "conv " + L.name + ": up-residual excludes other epilogue inputs");
    const bool flat = is_flat(L, io);
    conv_tiling(L, io, L.Cout_pad / block_n, cp);
    const int N = in.N, tw = 1 << cp->tw_log2, th = cp->th;
    // operand boxes: one tile's input pixels (flat: 128 consecutive pixels of the one-row view)
    auto a_map = [&](CUtensorMap* m, const Act& a, int s) {
        return flat ? make_act_map(h, m, a.ptr, a.C, cp->Wout, 1, 1, h->planes, a.plane(), 128, 1, 1)
                    : make_act_map(h, m, a.ptr, a.C, a.W, a.H, N, h->planes, a.plane(), tw * s, th * s, s);
    };
    int rc = a_map(&cp->tmA, in, L.stride);
    if (!rc && in2) rc = a_map(&cp->tmA2, *in2, L.stride2);
    if (rc) return rc;
    cp->Cout = L.Cout_pad;
    cp->kh = cp->kw = L.k;
    cp->stride = L.stride;
    cp->pad_y = cp->pad_x = L.pad;
    cp->kchunks = L.Cin / 64;
    cp->kchunks2 = L.Cin2 / 64;
    cp->stride2 = L.stride2;
    cp->bias = L.bias_dev;
    cp->has_res = (res || up) ? 1 : 0;
    cp->n_post = (post1 ? 1 : 0) + (post2 ? 1 : 0);
    if (up) {  // fused bilinear x2 residual: the ring carries the low-resolution patch under each output tile
        cp->up_mode = 1;
        cp->up_Hi = up->H;
        cp->up_Wi = up->W;
        cp->up_pw = tw / 2 + 2;
        cp->up_ph = th / 2 + 2;
        if (up->H * 2 != cp->Hout || up->W * 2 != cp->Wout || up->C != L.Cout_pad || cp->up_pw * cp->up_ph > 128)
            return fail(h, -30, "conv " + L.name + ": unsupported up-residual geometry");
        rc = make_act_map(h, &cp->tmR[0], up->ptr, up->C, up->W, up->H, N, h->planes, up->plane(), cp->up_pw,
                          cp->up_ph, 1, 32);
        if (rc) return rc;
    }
    if (post2 && !post1) return fail(h, -30, "conv " + L.name + ": post2 without post1");
    cp->out = io.out ? io.out->ptr : nullptr;
    cp->out_f32 = io.out_f32 ? io.out_f32->ptr : nullptr;
    cp->plane_stride = (long long)cp->Nimg * cp->Hout * cp->Wout * L.Cout_pad;
    cp->relu = io.relu;
    cp->sat = h->sat_dev;
    rc = make_w_map(h, &cp->tmB, L.w_dev, L.Cin + L.Cin2, L.Cout_pad, L.k * L.k, h->planes, block_n);
    if (rc) return rc;
    // epilogue tiles: 32 channels x (tw x th) pixels of the output / residual planes
    int n_in = up ? 1 : 0;
    for (const Act* t : {io.out, res, post1, post2}) {
        if (!t) continue;
        CUtensorMap* m = t == io.out ? &cp->tmO : &cp->tmR[n_in++];
        rc = make_act_map(h, m, t->ptr, L.Cout_pad, cp->Wout, cp->Hout, cp->Nimg, h->planes, t->plane(), tw, th, 1, 32);
        if (rc) return rc;
    }
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
    set_tiling(cp, N, H2, W2, patch_width(H2, W2, 1, false), 1);
    const long long WP = W2 + 3;
    cuuint64_t dims[5] = {64, (cuuint64_t)W2, (cuuint64_t)H2, (cuuint64_t)N, (cuuint64_t)h->planes};
    cuuint64_t strides[4] = {32, (cuuint64_t)WP * 32, (cuuint64_t)H2 * WP * 32, (cuuint64_t)s2d_plane * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)(1 << cp->tw_log2), (cuuint32_t)cp->th, 1, 1};
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(&cp->tmA, elem_dtype(h), 5, (void*)s2d, dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(h, -22, "sliding-window tensor map rejected: " + std::to_string((int)r));
    cp->Cout = 64;
    cp->kh = 4, cp->kw = 1, cp->stride = 1, cp->pad_y = 2, cp->pad_x = 0;
    cp->kchunks = 1;
    cp->bias = L.bias_dev;
    cp->out = out.ptr;
    cp->plane_stride = out.plane();
    cp->relu = 1;
    cp->sat = h->sat_dev;
    int rc = make_w_map(h, &cp->tmB, L.w_dev, 64, 64, 4, h->planes, 64);
    if (rc) return rc;
    rc = make_act_map(h, &cp->tmO, out.ptr, 64, W2, H2, N, h->planes, out.plane(), 1 << cp->tw_log2, cp->th, 1, 32);
    if (rc) return rc;
    *block_n_out = 64;
    *flops_out = 2.0 * N * H2 * W2 * 64.0 * 147.0;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// tile choice
// ------------------------------------------------------------------------------------------------
// A table row holds (BLOCK_N, CTAs per tile); a row this kernel has no variant for (a table written for another GPU) is
// measured again
bool table_row_ok(const std::pair<int, int>& row) { return row.second == 1 && tile_shape_ok(row.first); }

// The tile width of a plan conv from the process-wide table or, for a geometry it does not cover, from the autotuner: time
// every valid width once (activation contents do not matter for the timing), keep the fastest and add it to the table.
// Leaves *bn as it is when neither applies.
int table_tile(smapb_handle* h, const ConvLayer& L, const ConvIO& io, int* bn) {
    const Act& in = *io.in;
    char key[256];
    // fp16 rows carry the element type: they never match (or overwrite) a bf16 row of the same geometry.  (Cin2 appears
    // twice: the committed tables are keyed so.)
    snprintf(key, sizeof key, "%d/%d/%d k%d s%d %dx%dx%d r%d p%d u%d c2_%d s2_%d t%d%s", L.Cin, L.Cout_pad, L.Cin2, L.k,
             L.stride, in.N, in.H, in.W, io.res ? 1 : 0, (io.post1 ? 1 : 0) + (io.post2 ? 1 : 0), io.up ? 1 : 0, L.Cin2,
             L.stride2, h->nterms, h->f16 ? " f16" : "");
    {
        std::lock_guard<std::mutex> lk(g_tiles_mu);
        auto it = g_tiles.find(key);
        if (it != g_tiles.end() && table_row_ok(it->second)) {
            *bn = it->second.first;
            return 0;
        }
    }
    if (!h->autotune) return 0;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best_ms = 1e30f;
    int best = 0;
    for (int c : {128, 64, 32}) {
        if (L.Cout_pad % c) continue;
        if (c == 32 && L.Cout_pad > 64) continue;
        ConvParams trial;
        if (setup_conv(h, L, io, c, &trial)) continue;
        // trial launches run on the plan's zero-filled activations (output = bias): their clamps are not the
        // user's, so they stay out of the saturation counter (the kernel still clamps)
        trial.sat = nullptr;
        float ms_best_c = 1e30f;
        for (int rep = 0; rep < 4; rep++) {
            cudaEventRecord(e0, nullptr);
            if (launch_conv(trial, c, h->nterms, h->f16, h->sm_count, nullptr) != cudaSuccess) {
                ms_best_c = 1e30f;
                break;
            }
            cudaEventRecord(e1, nullptr);
            if (cudaEventSynchronize(e1) != cudaSuccess) return fail(h, -10, "autotune launch failed");
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            if (rep > 0 && ms < ms_best_c) ms_best_c = ms;
        }
        if (ms_best_c < best_ms) best_ms = ms_best_c, best = c;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    h->err.clear();
    if (!best) return 0;
    std::lock_guard<std::mutex> lk(g_tiles_mu);
    auto it = g_tiles.find(key);
    if (it == g_tiles.end() || !table_row_ok(it->second))
        g_tiles[key] = std::make_pair(best, 1);  // new, or replaces a row this kernel cannot run
    else
        best = it->second.first;  // another handle may have been first
    *bn = best;
    return 0;
}

// The tile width (BLOCK_N) of a conv.  Later rules override earlier ones:
//  1. a coarse cost model;
//  2. SMAPB_FORCE_TILE=<bn>, where the width divides the layer's padded output channels;
//  3. with `tuned` (the plan's convs with split outputs): the tile table's row, or the autotuner's winner.
int choose_tile(smapb_handle* h, const ConvLayer& L, const ConvIO& io, bool tuned, int* bn_out) {
    ConvParams tiling;
    conv_tiling(L, io, 1, &tiling);
    const long long m_tiles = tiling.total_tiles;
    // The cost model: a tile's main loop costs about num_kb x (relative wgmma time of a 128 x c tile) and every tile pays an
    // epilogue.  The two consumer warpgroups overlap one tile's epilogue with the next tile's main loop, but a CTA's last
    // epilogue and the epilogues of short-K tiles (epilogue longer than a main loop) stay exposed, so the model keeps
    // time ~ waves x (main loop + epilogue).  Near-ties go to the wider tile.  The model only decides geometries that
    // neither the committed tile table (smap_b200/tiles/h100.tsv, measured with this kernel by tools/make_tile_table.py)
    // nor the autotuner covers.
    int bn = 0;
    const int num_kb = L.k * L.k * (L.Cin / 64) + L.Cin2 / 64;
    double best = 1e30;
    for (int c : {128, 64, 32}) {
        if (L.Cout_pad % c) continue;
        const double kb_cost = c == 128 ? 1.0 : c == 64 ? 0.6 : 0.4;
        const int n_extra = (io.res || io.up ? 1 : 0) + (io.post1 ? 1 : 0) + (io.post2 ? 1 : 0);
        const double epi = (c / 32) * (0.5 + 0.2 * n_extra + (io.up ? 0.5 : 0.0));
        const long long units = m_tiles * (L.Cout_pad / c);
        const double waves = (double)((units + h->sm_count - 1) / h->sm_count);
        double t = waves * (num_kb * kb_cost + epi);
        t *= (c == 64 ? 1.05 : c == 32 ? 1.10 : 1.0);
        if (t < best - 1e-9) best = t, bn = c;
    }
    if (!bn) return fail(h, -30, "conv " + L.name + ": no tile shape for Cout_pad " + std::to_string(L.Cout_pad));
    if (const char* force = getenv("SMAPB_FORCE_TILE")) {  // debug
        int fb = 0;
        if (sscanf(force, "%d", &fb) == 1 && tile_shape_ok(fb) && L.Cout_pad % fb == 0) bn = fb;
    }
    if (tuned) {
        const int rc = table_tile(h, L, io, &bn);
        if (rc) return rc;
    }
    *bn_out = bn;
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

// wf holds [Cout][Cin + Cin2][taps] (taps == 1 for fused pairs)
int upload_conv_layer(smapb_handle* h, ConvLayer& L, int taps, const std::vector<float>& wf, const std::vector<float>& bf) {
    const int cin = L.Cin + L.Cin2;
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
    if (dev_alloc(h, L.w_dev, host.size()) || dev_alloc(h, L.bias_dev, bias.size())) return -10;
    CK(cudaMemcpy(L.w_dev, host.data(), host.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(L.bias_dev, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
    return 0;
}

int pad32(int c) { return (c + 31) / 32 * 32; }

bool precision_ok(int p) { return p == SMAPB_PREC_BF16X3 || p == SMAPB_PREC_BF16 || p == SMAPB_PREC_FP16; }
void set_precision(smapb_handle* h, int precision) {
    h->nterms = precision == SMAPB_PREC_BF16X3 ? 3 : 1;
    h->planes = precision == SMAPB_PREC_BF16X3 ? 2 : 1;
    h->f16 = precision == SMAPB_PREC_FP16;
}

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct PlanBuilder {
    smapb_handle* h;
    Plan* plan;
    int rc = 0;
    int cur_stream = 0;  // stream of the ops being added (0 main chain, 1 side branches)

    // record op (just pushed) as the producer of `out_ptr` and wire cross-stream waits for its inputs
    void wire(const void* out_ptr, const std::vector<const void*>& inputs) {
        const int idx = (int)plan->ops.size() - 1;
        Op& op = plan->ops[idx];
        op.stream = cur_stream;
        op.inputs = inputs;
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

    void* alloc(size_t bytes, const char* what) {
        DeviceBuffer<uint8_t> b;
        if (b.grow(bytes) != cudaSuccess) {
            rc = fail(h, -10, std::string("cudaMalloc failed for ") + what);
            return nullptr;
        }
        plan->allocs.push_back(std::move(b));
        return plan->allocs.back().get();
    }
    Act new_act(int N, int H, int W, int C) {
        Act a;
        a.N = N, a.H = H, a.W = W, a.C = C;
        a.ptr = (__nv_bfloat16*)alloc((size_t)a.plane() * 2 * h->planes, "activation tensor");
        // one-time zero fill: every element is overwritten by its producer before it is read, but the producers store
        // through TMA (cp.async.bulk.tensor), which compute-sanitizer's initcheck does not track
        if (a.ptr) cudaMemset(a.ptr, 0, (size_t)a.plane() * 2 * h->planes);
        return a;
    }
    ActF32 new_f32(int N, int H, int W, int C) {
        ActF32 a;
        a.N = N, a.H = H, a.W = W, a.C = C;
        a.ptr = (float*)alloc((size_t)N * H * W * C * 4, "fp32 tensor");
        return a;
    }
    const ConvLayer* layer(const std::string& name) {
        auto it = h->layers.find(name);
        if (it == h->layers.end()) {
            rc = fail(h, -41, "layer not found: " + name);
            return nullptr;
        }
        return &it->second;
    }
    // Adds conv `name` over io's inputs; it writes a new split tensor (returned), or a new fp32 tensor into *f32 (the heads).
    // Only split-output convs take their tile width from the tile table or the autotuner.
    Act conv(const std::string& name, ConvIO io, ActF32* f32 = nullptr) {
        Act out;
        if (rc) return out;
        const ConvLayer* L = layer(name);
        if (!L) return out;
        const Act& in = *io.in;
        const int Ho = (in.H + 2 * L->pad - L->k) / L->stride + 1, Wo = (in.W + 2 * L->pad - L->k) / L->stride + 1;
        if (f32) {
            *f32 = new_f32(in.N, Ho, Wo, L->Cout_pad);
            io.out_f32 = f32;
        } else {
            out = new_act(in.N, Ho, Wo, L->Cout_pad);
            io.out = &out;
        }
        if (rc) return out;
        Op op;
        op.kind = OP_CONV;
        rc = choose_tile(h, *L, io, !f32, &op.block_n);
        if (!rc) rc = setup_conv(h, *L, io, op.block_n, &op.cp);
        op.flops = 2.0 * in.N * Ho * Wo * (double)L->Cout * (L->Cin * L->k * L->k + L->Cin2);
        op.name = name;
        op.dims[0] = in.N, op.dims[1] = Ho, op.dims[2] = Wo, op.dims[3] = L->Cout_pad;
        plan->ops.push_back(op);
        wire(f32 ? (const void*)f32->ptr : out.ptr, io.inputs());
        plan->n_conv++;
        plan->conv_flops += op.flops;
        return out;
    }
};

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
    const bool is_conv = op.kind == OP_CONV;
    const bool stem_tc = is_conv && op.cp.kh == 4 && op.cp.kw == 1;
    const char* kind = is_conv ? (stem_tc ? "stem_tc" : op.cp.out ? "conv" : "conv_f32")
                       : op.kind == OP_STEM ? "stem" : op.kind == OP_S2D ? "s2d" : op.kind == OP_MAXPOOL ? "maxpool"
                       : "other";
    std::string s = "name=" + (op.name.empty() ? std::string("?") : op.name) + " kind=" + kind;
    if (op.kind == OP_STEM || op.kind == OP_S2D) s += " in=x";  // the network input image
    for (size_t r = 0; r < op.inputs.size(); r++) {
        if (!op.inputs[r]) continue;
        const char* role = is_conv ? (r < 6 ? CONV_ROLES[r] : "?") : "a";
        auto it = dump_idx.find(op.inputs[r]);
        s += std::string(" ") + role + "=" + (it == dump_idx.end() ? std::string("?") : std::to_string(it->second));
    }
    char buf[320];
    if (is_conv) {
        snprintf(buf, sizeof buf,
                 " tw=%d k=%dx%d s=%d pad=%dx%d cin=%d cin2=%d s2=%d cout=%d out=%dx%dx%dx%d bn=%d relu=%d "
                 "hasres=%d post=%d upmode=%d tiles=%d nterms=%d",
                 1 << op.cp.tw_log2, op.cp.kh, op.cp.kw, op.cp.stride, op.cp.pad_y, op.cp.pad_x,
                 op.cp.kchunks * 64, op.cp.kchunks2 * 64, op.cp.stride2, op.cp.Cout, op.dims[0], op.dims[1], op.dims[2],
                 op.dims[3], op.block_n, op.cp.relu, op.cp.has_res, op.cp.n_post, op.cp.up_mode, op.cp.total_tiles,
                 h->nterms);
    } else {
        snprintf(buf, sizeof buf, " out=%dx%dx%dx%d nterms=%d", op.out.N, op.out.H, op.out.W, op.out.C, h->nterms);
    }
    return s + buf + (h->f16 ? " dtype=f16" : "");
}

}  // namespace

namespace smapb {

int build_plan(smapb_handle* h, int B, Plan** out_plan) {
    auto it = h->plans.find(B);
    if (it != h->plans.end()) {
        *out_plan = it->second.get();
        return 0;
    }
    std::unique_ptr<Plan> plan(new Plan());
    plan->B = B;
    PlanBuilder pb{h, plan.get()};
    const int H = h->in_h, W = h->in_w;
    static const int LAYERS[4] = {3, 4, 6, 3};
    // stem + maxpool (model/smap.py:88-92)
    Act stem = pb.new_act(B, H / 2, W / 2, 64);
    {
        // tensor-core stem over the space-to-depth input when the driver accepts the sliding-window TMA view,
        // otherwise the fp32 CUDA-core stem kernel (both are GPU paths; SMAPB_STEM=cuda forces the latter)
        bool tc = h->stem_tc_ok != 0 && !(getenv("SMAPB_STEM") && !strcmp(getenv("SMAPB_STEM"), "cuda"));
        if (tc) {
            const Act s2d = pb.new_act(B, H / 2, W / 2 + 3, 16);  // storage [plane][B][H/2][W/2+3][16]
            if (pb.rc) return pb.rc;
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
                Act o1 = pb.conv(p + "conv_bn_relu1", {&t, 1});
                Act o2 = pb.conv(p + "conv_bn_relu2", {&o1, 1});
                const bool last = (b == LAYERS[li] - 1) && s > 0;
                ConvIO c3{&o2, 1};
                if (b == 0) {
                    // relu(conv3(o2) + downsample(x)) as one K-concatenated GEMM
                    c3.in2 = &t;
                    t = pb.conv(p + "fused_conv3_downsample", c3);
                } else {
                    // out = relu(conv3 + x) [ + skip1 + skip2 ]   (model/smap.py:74-75,143)
                    c3.res = &t;
                    if (last) c3.post1 = &skip1[li], c3.post2 = &skip2[li];
                    t = pb.conv(p + "conv_bn_relu3", c3);
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
                out = pb.conv(p + "u_skip", {&xin, 1});
            } else {
                // out = relu(u_skip(x) + bilinear_x2(up_conv(up_x))): the 1x1 up_conv is commuted in front of the
                // interpolation (both linear, bilinear weights sum to 1) and the interpolation + add + ReLU run in the
                // u_skip epilogue
                Act tl = pb.conv(p + "up_conv", {&up_x, 0});
                ConvIO io{&xin, 1};
                io.up = &tl;
                out = pb.conv(p + "u_skip", io);
            }
            // Side branches (heads, skip convs) hang off `out` / `xin` and are only needed much later: they go to the
            // second stream and overlap the main chain, filling SMs that small layers leave idle.
            pb.cur_stream = 1;
            // heads: only those that reach the returned tensors (model/smap.py:418-419) are computed
            if (s == 2 && ind >= 1) {
                Act r1 = pb.conv(p + "res_conv1", {&out, 1});
                pb.conv(p + "res_conv2", {&r1, 0}, &res[ind]);
            }
            if (s == 2 && ind == 3) {
                Act d1 = pb.conv(p + "res_d_conv1", {&out, 1});
                pb.conv(p + "res_d_conv2.tapexp", {&d1, 0}, &resd3);
                Act rd1 = pb.conv(p + "res_rd_conv1", {&out, 1});
                pb.conv(p + "res_rd_conv2.tapexp", {&rd1, 0}, &resrd3);
                name_d = p + "res_d_conv2";
                name_rd = p + "res_rd_conv2";
            }
            if (gen_skip) {
                sk1[ind] = pb.conv(p + "skip1", {&xin, 1});
                sk2[ind] = pb.conv(p + "skip2", {&out, 1});
                pb.cur_stream = 0;
                if (ind == 3) cross = pb.conv(p + "cross_conv", {&out, 1});
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
    if (pb.rc) return pb.rc;
    {
        Op op;
        op.kind = OP_HEADMERGE;
        op.name = "head_merge(res4+res3+res2)";
        op.f4 = res[3], op.f3 = res[2], op.f2 = res[1];
        op.cout = 43;
        plan->ops.push_back(op);
        pb.wire(nullptr, {res[3].ptr, res[2].ptr, res[1].ptr});
        for (int which = 1; which <= 2; which++) {  // the depth heads' tap sums: 1 detd (14 channels), 2 rootd (1)
            Op od;
            od.kind = OP_TAPSUM;
            od.name = which == 1 ? "tapsum(res_d)" : "tapsum(res_rd)";
            od.f4 = which == 1 ? resd3 : resrd3;
            od.cout = which == 1 ? 14 : 1;
            od.which_out = which;
            od.bias = h->layers[which == 1 ? name_d : name_rd].bias_dev;
            plan->ops.push_back(od);
            pb.wire(nullptr, {od.f4.ptr});
        }
        // the main stream must not run ahead of the side stream into the next forward: the last op joins it
        if (plan->last_side >= 0) {
            plan->ops[plan->last_side].record = true;
            plan->ops.back().waits.push_back(plan->last_side);
        }
    }
    for (Op& op : plan->ops)
        if (op.record) cudaEventCreateWithFlags(&op.ev, cudaEventDisableTiming);
    *out_plan = plan.get();
    h->plans[B] = std::move(plan);
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
        const NvtxScope range(op.name.empty() ? "smapb.op" : op.name.c_str(), h->nvtx_ops);
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
                    CK(launch_conv(cp, op.block_n, h->nterms, h->f16, h->sm_count, st));
                } else {
                    CK(launch_conv(op.cp, op.block_n, h->nterms, h->f16, h->sm_count, st));
                }
                if (h->profiling) {
                    char d[160];
                    snprintf(d, sizeof d, "conv k%dx%d s%d cin%d cout%d out%dx%d bn%d tiles%d", op.cp.kh, op.cp.kw,
                             op.cp.stride, op.cp.kchunks * 64, op.cp.Cout, op.cp.Hout, op.cp.Wout, op.block_n,
                             op.cp.total_tiles);
                    prof_mark(h, PK_CONV, st, d, op.flops);
                    if (h->roles_dev) h->roles_desc.push_back(op.name + "," + d);
                }
                break;
            case OP_TAPSUM: {
                float* dst = op.which_out == 1 ? detd : rootd;
                CK(launch_tapsum(op.f4.ptr, op.bias, B, op.f4.H, op.f4.W, op.f4.C, op.cout, dst, st));
                prof_mark(h, PK_ELEM, st, "tapsum");
                break;
            }
            case OP_HEADMERGE:
                CK(launch_head_merge(op.f4.ptr, op.f3.ptr, op.f2.ptr, B, op.f4.H, op.f4.W, op.f3.H, op.f3.W, op.f2.H,
                                     op.f2.W, op.f4.C, op.cout, hm2d, st));
                prof_mark(h, PK_ELEM, st, "head_merge");
                break;
        }
        h->launches++;
        if (multi && op.record) CK(cudaEventRecord(op.ev, st));
        static const bool debug_sync = getenv("SMAPB_DEBUG_SYNC") != nullptr;
        if (debug_sync) CK(cudaStreamSynchronize(st));
    }
    return 0;
}

}  // namespace smapb

// ================================================================================================
// C ABI: weights, tile table, plan introspection, conv test hook
// ================================================================================================
extern "C" {
#pragma GCC visibility push(default)

int smapb_finalize_weights(smapb_handle* h, int precision) {
    if (!h) return -1;
    if (!precision_ok(precision)) return fail(h, -1, "unknown precision");
    cudaSetDevice(h->device);
    // a new weight set invalidates cached plans (they hold tensor maps over the old weight buffers only if
    // buffers are re-allocated; buffers are reused in place, but the plane count may change)
    const int new_planes = precision == SMAPB_PREC_BF16X3 ? 2 : 1;
    h->finalized = false;
    drop_graphs(h);
    h->eager_runs.clear();
    if (new_planes != h->planes || !h->plans.empty()) {
        cudaDeviceSynchronize();
        h->plans.clear();
        h->layers.clear();
        h->stem_tc = ConvLayer();
    }
    set_precision(h, precision);
    // unit names: every "<name>.conv.weight" key
    std::vector<std::string> units;
    for (auto& kv : h->raw) {
        const std::string& k = kv.first;
        const std::string suf = ".conv.weight";
        if (k.size() > suf.size() && k.compare(k.size() - suf.size(), suf.size(), suf) == 0)
            units.push_back(k.substr(0, k.size() - suf.size()));
    }
    if (units.empty()) return fail(h, -40, "no weights loaded");
    struct Folded {
        ConvGeom L;
        std::vector<float> w, b;
    };
    std::map<std::string, Folded> folded;  // units the loops below build other layers from
    for (const std::string& name : units) {
        std::vector<float> wf, bf;
        int Cout, Cin, k;
        int rc = fold_unit(h, name, &wf, &bf, &Cout, &Cin, &k);
        if (rc) return rc;
        // conv3 and downsample of a layer's first bottleneck: the plan only runs them as their fused pair
        const bool pair_half = name.find(".downsample.layer") != std::string::npos &&
                               (name.find(".0.conv_bn_relu3") != std::string::npos ||
                                (name.size() > 13 && name.compare(name.size() - 13, 13, ".0.downsample") == 0));
        if (name == "top.conv") {
            if (Cin != 3 || Cout != 64 || k != 7) return fail(h, -40, "top.conv must be 3->64 7x7");
            std::vector<float> w2(147 * 64);
            for (int co = 0; co < 64; co++)
                for (int ci = 0; ci < 3; ci++)
                    for (int ky = 0; ky < 7; ky++)
                        for (int kx = 0; kx < 7; kx++)
                            w2[((ky * 7 + kx) * 3 + ci) * 64 + co] = wf[((co * 3 + ci) * 7 + ky) * 7 + kx];
            if (dev_alloc(h, h->stem_w, w2.size()) || dev_alloc(h, h->stem_b, 64)) return -10;
            CK(cudaMemcpy(h->stem_w, w2.data(), w2.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(h->stem_b, bf.data(), 64 * 4, cudaMemcpyHostToDevice));
            // tensor-core stem: 4 taps (ky-blocks ay) of 64 k = ax*16 + (by*2+bx)*3 + c; ky = 2*ay+by-1, kx = 2*ax+bx-1
            ConvLayer& S = h->stem_tc;
            S.name = name;
            S.Cin = 64, S.Cout = 64, S.Cout_pad = 64;
            std::vector<float> ws((size_t)64 * 64 * 4, 0.f);
            for (int co = 0; co < 64; co++)
                for (int ay = 0; ay < 4; ay++)
                    for (int ax = 0; ax < 4; ax++)
                        for (int by = 0; by < 2; by++)
                            for (int bx = 0; bx < 2; bx++)
                                for (int c = 0; c < 3; c++) {
                                    const int ky = 2 * ay + by - 1, kx = 2 * ax + bx - 1;
                                    if (ky < 0 || ky > 6 || kx < 0 || kx > 6) continue;
                                    ws[((size_t)co * 64 + ax * 16 + (by * 2 + bx) * 3 + c) * 4 + ay] =
                                        wf[((co * 3 + c) * 7 + ky) * 7 + kx];
                                }
            rc = upload_conv_layer(h, S, 4, ws, bf);
            if (rc) return rc;
            continue;
        }
        ConvLayer unit;
        ConvLayer& L = pair_half ? unit : h->layers[name];
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
                const int blk = atoi(name.c_str() + pl + 19);
                const bool first = blk == 0;
                const bool is_c2 = name.find("conv_bn_relu2") != std::string::npos;
                const bool is_ds = name.size() > 11 && name.compare(name.size() - 11, 11, ".downsample") == 0;
                if (li >= 2 && first && (is_c2 || is_ds)) L.stride = 2;
            }
        }
        if (pair_half) {
            if (h->f16 && check_f16_range(h, name, wf.data(), wf.size())) return -42;
            folded[name] = {L, std::move(wf), std::move(bf)};
            continue;
        }
        if (name.find("res_d_conv2") != std::string::npos || name.find("res_rd_conv2") != std::string::npos)
            folded[name] = {L, wf, bf};
        int rc2 = upload_conv_layer(h, L, k * k, wf, bf);
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
        const ConvGeom& L3 = kv.second.L;
        const ConvGeom& Lds = ids->second.L;
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
            for (int ci = 0; ci < F.Cin; ci++) wf[(size_t)co * cin + ci] = kv.second.w[(size_t)co * F.Cin + ci];
            for (int ci = 0; ci < F.Cin2; ci++) wf[(size_t)co * cin + F.Cin + ci] = ids->second.w[(size_t)co * F.Cin2 + ci];
            bf[co] = kv.second.b[co] + ids->second.b[co];
        }
        int rc3 = upload_conv_layer(h, F, 1, wf, bf);
        if (rc3) return rc3;
    }
    // thin 3x3 heads as tap expansion: rows (tap*C + c) of a 1x1 GEMM, bias applied by the gather kernel
    for (auto& kv : folded) {
        const std::string& nm = kv.first;
        if (nm.find("res_d_conv2") == std::string::npos && nm.find("res_rd_conv2") == std::string::npos) continue;
        const ConvGeom& L0 = kv.second.L;
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
                    wf[(size_t)(t * L0.Cout + c) * E.Cin + ci] = kv.second.w[((size_t)c * L0.Cin + ci) * 9 + t];
        int rc4 = upload_conv_layer(h, E, 1, wf, bf);
        if (rc4) return rc4;
    }
    if (!h->stem_w) return fail(h, -40, "top.conv weights missing");
    h->finalized = true;
    return 0;
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
        int bn = 0, ctas = 1;
        if (sscanf(line.c_str() + t1 + 1, "%d\t%d", &bn, &ctas) < 1 || bn <= 0) continue;
        g_tiles[line.substr(0, t1)] = {bn, ctas};
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
    DeviceBuffer<unsigned long long> d;
    CK(d.grow(1));
    std::map<const void*, int> dump_idx;  // output tensor -> dump index (the numbering of smapb_debug_dump)
    int n_dumped = 0;
    for (const Op& op : plan->ops) {
        long long bytes = 0;
        const void* out = dumped_output(h, op, &bytes);
        if (!out) continue;
        if (!dump_idx.emplace(out, n_dumped++).second)
            return fail(h, -2, "smapb_debug_checksums: two ops share an output tensor (" + op.name + ")");
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
    return n;
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
                    const float* post1, const float* post2, const float* in2_src, const float* up_src, int B, int H, int W,
                    int Cin, int Cout, int k, int stride, int H2, int W2, int Cin2, int stride2, int relu, int out_f32,
                    int precision, float* y, int* launch, float* ms_out, void* stream) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (!precision_ok(precision)) return fail(h, -1, "smapb_conv_test: unknown precision");
    if (B < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || k < 1 || stride < 1 || Cin2 < 0)
        return fail(h, -1, "smapb_conv_test: bad geometry");
    const int pad = k / 2;
    const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    if (in2_src && (stride2 < 1 || H2 < 1 || W2 < 1 || (H2 - 1) / stride2 + 1 != Ho || (W2 - 1) / stride2 + 1 != Wo))
        return fail(h, -1, "smapb_conv_test: in2 does not give the output geometry under stride2");
    struct RestorePrecision {  // the handle's precision, put back on every return
        smapb_handle* h;
        int nterms, planes;
        bool f16;
        ~RestorePrecision() { h->nterms = nterms, h->planes = planes, h->f16 = f16; }
    } restore{h, h->nterms, h->planes, h->f16};
    set_precision(h, precision);
    int rc = 0;
    ConvLayer L;
    L.name = "conv_test";
    L.Cin = Cin, L.Cout = Cout, L.Cout_pad = pad32(Cout), L.k = k, L.stride = stride, L.pad = pad;
    L.Cin2 = Cin2, L.stride2 = stride2;
    std::vector<float> wh((size_t)Cout * (Cin + Cin2) * k * k), bh(Cout);
    CK(cudaMemcpy(wh.data(), w, wh.size() * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(bh.data(), bias, bh.size() * 4, cudaMemcpyDeviceToHost));
    rc = upload_conv_layer(h, L, k * k, wh, bh);
    if (rc) return rc;
    Act in, out, in2, up;
    ActF32 out32;
    in.N = B, in.H = H, in.W = W, in.C = Cin;
    out.N = B, out.H = Ho, out.W = Wo, out.C = L.Cout_pad;
    in2.N = B, in2.H = H2, in2.W = W2, in2.C = Cin2;
    up.N = B, up.H = Ho / 2, up.W = Wo / 2, up.C = Cout;
    out32.N = B, out32.H = Ho, out32.W = Wo, out32.C = L.Cout_pad;
    ConvIO io{&in, relu};
    DeviceBuffer<__nv_bfloat16> in_buf, in2_buf, out_buf, extra_buf[4];
    DeviceBuffer<float> y32;  // the fp32 output: the conv's own (out_f32), or its split output converted
    // the operands in the precision's activation planes, converted as the plan converts fp32 tensors (an empty tensor,
    // an in2 with Cin2 = 0 or an up of a 1-pixel output, is left unallocated: setup_conv refuses it)
    auto planes_of = [&](const float* src, Act& a, DeviceBuffer<__nv_bfloat16>& buf) -> cudaError_t {
        if (a.plane() == 0) return cudaSuccess;
        cudaError_t e = buf.grow((size_t)a.plane() * h->planes);
        if (e != cudaSuccess) return e;
        a.ptr = buf;
        return launch_f32_to_split(src, a.ptr, a.plane(), a.plane(), h->planes, st, h->f16);
    };
    CK(planes_of(x, in, in_buf));
    if (out_f32) {
        CK(y32.grow((size_t)out.plane()));
        out32.ptr = y32;
        CK(cudaMemset(y32, 0, (size_t)out.plane() * 4));
        io.out_f32 = &out32;
    } else {
        CK(out_buf.grow((size_t)out.plane() * h->planes));
        out.ptr = out_buf;
        CK(cudaMemset(out_buf, 0, (size_t)out.plane() * 2 * h->planes));  // TMA stores are invisible to initcheck
        io.out = &out;
    }
    if (in2_src) {
        CK(planes_of(in2_src, in2, in2_buf));
        io.in2 = &in2;
    }
    const float* extra_src[4] = {res, post1, post2, up_src};
    Act extra_act[4] = {out, out, out, up};
    const Act** extra_role[4] = {&io.res, &io.post1, &io.post2, &io.up};
    for (int e = 0; e < 4; e++) {
        if (!extra_src[e]) continue;
        if (L.Cout_pad != Cout) return fail(h, -1, "conv_test: residual/post/up operands require Cout % 32 == 0");
        CK(planes_of(extra_src[e], extra_act[e], extra_buf[e]));
        *extra_role[e] = &extra_act[e];
    }
    ConvParams cp;
    int bn = 0;
    rc = choose_tile(h, L, io, false, &bn);
    if (!rc) rc = setup_conv(h, L, io, bn, &cp);
    if (rc) return rc;
    if (launch) {
        launch[0] = bn;
        launch[1] = 1 << cp.tw_log2;
        launch[2] = is_flat(L, io) ? 1 : 0;
        launch[3] = conv_ring(cp);
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    DeviceBuffer<long long> dbg_dev, tl_dev;
    if (getenv("SMAPB_ROLES")) {
        CK(dbg_dev.grow(16));
        CK(cudaMemset(dbg_dev, 0, 16 * sizeof(long long)));
        cp.dbg = dbg_dev;
    }
    if (getenv("SMAPB_TIMELINE")) CK(tl_dev.grow(16));
    CK(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st));  // warm-up + result
    cp.sat = nullptr;  // the saturation counter counts the result launch; the time-line and timed re-runs leave it alone
    if (dbg_dev) {
        long long d[16];
        CK(cudaMemcpy(d, dbg_dev, sizeof d, cudaMemcpyDeviceToHost));
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
        CK(cudaMemset(tl_dev, 0, 16 * sizeof(long long)));
        cp.dbg_tl = tl_dev;
        CK(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st));
        cp.dbg_tl = nullptr;
        long long t[16];
        CK(cudaMemcpy(t, tl_dev, sizeof t, cudaMemcpyDeviceToHost));
        fprintf(stderr, "[timeline] bn%d units%d kb%d | set-up %lld | first operands %lld | last main loop end %lld | epilogue done "
                "%lld | exit %lld\n", bn, cp.total_tiles, cp.kh * cp.kw * cp.kchunks + cp.kchunks2, t[1] - t[0], t[2] - t[0],
                t[3] - t[0], t[13] - t[0], t[15] - t[0]);
    }
    const int reps = ms_out ? 5 : 0;
    cudaEventRecord(e0, st);
    for (int i = 0; i < reps; i++) CK(launch_conv(cp, bn, h->nterms, h->f16, h->sm_count, st));
    cudaEventRecord(e1, st);
    h->launches += 1 + reps;
    // convert (split outputs) + de-pad
    if (!out_f32) {
        CK(y32.grow((size_t)out.plane()));
        split_to_f32_kernel<<<(unsigned)((out.plane() + 255) / 256), 256, 0, st>>>(out.ptr, out.plane(), h->planes, y32,
                                                                                   out.plane(), h->f16);
        CK(cudaGetLastError());
    }
    CK(cudaMemcpy2DAsync(y, (size_t)Cout * 4, y32, (size_t)L.Cout_pad * 4, (size_t)Cout * 4, (size_t)B * Ho * Wo,
                          cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    if (ms_out) {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        *ms_out = ms / reps;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return 0;
}

#pragma GCC visibility pop
}  // extern "C"
