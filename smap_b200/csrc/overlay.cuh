// The composite both image encoders write (jpeg_enc.cu, png_enc.cu): each frame with its skeleton overlay and, with
// SMAPB_ENCODE_VIEW3D, its 3D panel on the right (view3d.cu).  One stage owns the decision of which pixel shows what:
// the argument checks, the per-frame set-up from the scale rows, the label planes (overlay.cu) and load_pixel, the colour
// of one composite pixel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/smap_b200.h"
#include "decode_host.h"
#include "paint.cuh"
#include "view3d.h"

namespace smapb {

constexpr int NELEM = SMAPB_NL + SMAPB_NJ;  // 14 limbs then 15 joints per person: paint rank person * 29 + element + 1

// BGR limb colours per person (cycling), and the joint colour (include/smap_b200.h, smapb_encode_jpeg)
static __constant__ uint8_t kPalette[6][3] = {{0, 0, 255}, {0, 255, 0}, {255, 0, 0}, {0, 255, 255}, {0, 0, 0}, {255, 0, 255}};
static __constant__ uint8_t kJoint[3] = {255, 255, 255};
// the 3D panel's background and fit-box colour
static __constant__ uint8_t kWhite[3] = {255, 255, 255};
static __constant__ uint8_t kGrey[3] = {160, 160, 160};

// One composite image.
struct Composite {
    const uint8_t* src;  // BGR [h][fw][3]
    const smapb_record* rec;  // NULL: no overlay
    int h, w;  // the composite's size
    int fw;  // the frame's width: w, or w - h with the 3D panel in columns fw..w-1
    int r, R;  // limb half-width and joint radius (overlay)
    int pad_l, pad_t;  // letterbox of the net input (make_resize_plan)
    double scale;
    long long label0;  // first label of the image's plane [h][w] (overlay only; the panel's labels from column fw)
};

// The label planes of one call and the 3D panels' scratch, grown on demand.
struct CompositeStage {
    PinnedBuffer<double> scales_host;
    DeviceBuffer<int> labels;
    DeviceBuffer<PanelSeg> segs;  // [n][PANEL_ELEMS] (3D panel)
    std::vector<Composite> imgs;
    std::vector<PanelImg> panels;
    long long label_total = 0;
};

// The checks of an encoder call that come before its own (call names the entry point, call_ex its _ex variant): -1 with
// the text in *err for a null argument, unknown flags, or SMAPB_ENCODE_VIEW3D without records.
int composite_args(const char* call, const char* call_ex, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                   const smapb_record* records, const double* scales, int flags, std::string* err);

// The per-frame checks: a null frame, sides outside 1..16384, a composite wider than 16384.
int composite_frames(const char* call, const char* call_ex, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                     int flags, std::string* err);

// Copies the scale rows to the host (records only) and synchronises `st`; then fills cs->imgs, cs->panels and
// cs->label_total, or returns -1 when a scale row does not describe its frame.  Grows the label planes.
int composite_plan(CompositeStage* cs, const char* call, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                   const smapb_record* records, const double* scales, int flags, cudaStream_t st, std::string* err);

// The BGR colour of composite pixel (x, y): the frame's pixel or, where a label covers it, its element's colour; in the
// panel's columns white or the colour of the element painted last.
__device__ __forceinline__ void load_pixel(const Composite& I, const int* __restrict__ labels, int x, int y, int* b, int* g, int* r) {
    const size_t i = (size_t)y * I.w + x;
    const uint8_t* c = nullptr;
    if (x >= I.fw) {  // the 3D panel: white, or its element's colour (view3d.h)
        const int l = labels[I.label0 + i];
        c = l == 0 ? kWhite : (l & 7) == PANEL_GREY ? kGrey : kPalette[l & 7];
    } else {
        const uint8_t* s = I.src + ((size_t)y * I.fw + x) * 3;
        *b = s[0], *g = s[1], *r = s[2];
        if (I.rec) {
            const int l = labels[I.label0 + i];
            if (l > 0) {
                const int e = (l - 1) % NELEM, p = (l - 1) / NELEM;
                c = e < SMAPB_NL ? kPalette[p % 6] : kJoint;
            }
        }
    }
    if (c) *b = c[0], *g = c[1], *r = c[2];
}

// ---- overlay: one CTA per skeleton element walks a band around it and atomicMax-es its paint rank into the label plane,
// so the painter's order comes out whatever order the elements run in.  Compiled into each encoder.
namespace {

__device__ __forceinline__ bool joint_xy(const Composite& I, const float* pj, long long* x, long long* y) {
    if (!(pj[3] > 0.f) || !isfinite(pj[0]) || !isfinite(pj[1])) return false;
    const double fx = rint(((double)pj[0] - I.pad_l) / I.scale), fy = rint(((double)pj[1] - I.pad_t) / I.scale);
    *x = (long long)fmin(fmax(fx, (double)-COORD_MAX), (double)COORD_MAX);
    *y = (long long)fmin(fmax(fy, (double)-COORD_MAX), (double)COORD_MAX);
    return true;
}

__global__ void __launch_bounds__(256) overlay_kernel(const Composite* __restrict__ imgs, int* __restrict__ labels) {
    const Composite& I = imgs[blockIdx.y];
    if (!I.rec) return;
    const int p = blockIdx.x / NELEM, e = blockIdx.x % NELEM;
    if (p >= I.rec->count) return;
    const float* P = &I.rec->pred2d[p][0][0];
    long long ax, ay, bx, by, rad;
    if (e < SMAPB_NL) {
        if (!joint_xy(I, P + 4 * kPairs[e][0], &ax, &ay) || !joint_xy(I, P + 4 * kPairs[e][1], &bx, &by)) return;
        rad = I.r;
    } else {
        if (!joint_xy(I, P + 4 * (e - SMAPB_NL), &ax, &ay)) return;
        bx = ax, by = ay, rad = I.R;
    }
    // the frame's columns only: with a 3D panel the label plane is as wide as the composite
    paint_band(labels + I.label0, I.w, I.fw, I.h, ax, ay, bx, by, rad, p * NELEM + e + 1);
}

}  // namespace

// Clears the label planes and paints them: the overlay, then the 3D panels.  d_imgs / d_panels: device copies of cs->imgs /
// cs->panels.  Nothing is launched without records.  *launches counts the kernels; the caller checks cudaGetLastError.
inline int composite_launch(CompositeStage* cs, const Composite* d_imgs, const PanelImg* d_panels, int n, cudaStream_t st,
                     int64_t* launches, std::string* err) {
    if (!cs->label_total) return 0;
    DECODE_CK(cudaMemsetAsync(cs->labels, 0, sizeof(int) * cs->label_total, st));
    overlay_kernel<<<dim3(SMAPB_MAXP * NELEM, n), 256, 0, st>>>(d_imgs, cs->labels);
    ++*launches;
    if (!cs->panels.empty()) {
        panel_launch(d_panels, n, cs->segs, cs->labels, st);
        *launches += 2;
    }
    return 0;
}

}  // namespace smapb
