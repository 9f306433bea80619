// The composite stage of the image encoders (overlay.cuh): argument checks and per-frame set-up.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "overlay.cuh"
#include "preprocess.h"

namespace smapb {

int composite_args(const char* call, const char* call_ex, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                   const smapb_record* records, const double* scales, int flags, std::string* err) {
    if (n < 0 || (n > 0 && (!bgr || !img_h || !img_w)) || (records && !scales)) {
        *err = std::string(call) + ": null argument";
        return -1;
    }
    if (flags & ~SMAPB_ENCODE_VIEW3D) {
        *err = std::string(call_ex) + ": unknown flags " + std::to_string(flags);
        return -1;
    }
    if ((flags & SMAPB_ENCODE_VIEW3D) && !records) {
        *err = std::string(call_ex) + ": SMAPB_ENCODE_VIEW3D needs records";
        return -1;
    }
    return 0;
}

int composite_frames(const char* call, const char* call_ex, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                     int flags, std::string* err) {
    for (int i = 0; i < n; i++) {
        if (!bgr[i]) {
            *err = std::string(call) + ": null frame " + std::to_string(i);
            return -1;
        }
        if (img_h[i] < 1 || img_h[i] > 16384 || img_w[i] < 1 || img_w[i] > 16384) {
            *err = std::string(call) + ": frame " + std::to_string(i) + " is " + std::to_string(img_w[i]) + "x" +
                   std::to_string(img_h[i]) + " (sides must be 1..16384)";
            return -1;
        }
        if ((flags & SMAPB_ENCODE_VIEW3D) && img_w[i] + img_h[i] > 16384) {
            *err = std::string(call_ex) + ": frame " + std::to_string(i) + " is " + std::to_string(img_w[i]) + "x" +
                   std::to_string(img_h[i]) + ": with its 3D panel it would be " + std::to_string(img_w[i] + img_h[i]) +
                   " wide (sides must be 1..16384)";
            return -1;
        }
    }
    return 0;
}

int composite_plan(CompositeStage* cs, const char* call, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
                   const smapb_record* records, const double* scales, int flags, cudaStream_t st, std::string* err) {
    const bool view3d = flags & SMAPB_ENCODE_VIEW3D;
    if (records) {  // the letterbox of each frame, from its scale row
        DECODE_CK(cs->scales_host.grow((size_t)n * SMAPB_SCALE_LEN));
        DECODE_CK(cudaMemcpyAsync(cs->scales_host, scales, sizeof(double) * n * SMAPB_SCALE_LEN, cudaMemcpyDeviceToHost, st));
    }
    DECODE_CK(cudaStreamSynchronize(st));  // the scales, and the workspace the previous call may still use
    cs->imgs.assign(n, Composite{});
    cs->panels.assign(view3d ? n : 0, PanelImg{});
    long long label_total = 0;
    for (int i = 0; i < n; i++) {
        Composite& I = cs->imgs[i];
        memset(&I, 0, sizeof(I));
        I.src = bgr[i];
        I.h = img_h[i], I.fw = img_w[i];
        I.w = view3d ? I.fw + I.h : I.fw;
        I.label0 = -1;
        if (records) {
            const double* row = cs->scales_host + (size_t)i * SMAPB_SCALE_LEN;
            ResizePlan P;
            if (row[1] != I.fw || row[2] != I.h || !make_resize_plan(I.fw, I.h, (int)row[3], (int)row[4], &P)) {
                *err = std::string(call) + ": the scale row of frame " + std::to_string(i) + " does not describe a " +
                       std::to_string(I.fw) + "x" + std::to_string(I.h) + " frame";
                return -1;
            }
            I.rec = records + i;
            I.scale = row[0], I.pad_l = P.pad_l, I.pad_t = P.pad_t;
            const int m = std::min(I.fw, I.h);
            I.r = std::max(1, m / 400), I.R = std::max(2, m / 200);
            I.label0 = label_total;
            label_total += (long long)I.w * I.h;
            if (view3d) cs->panels[i] = PanelImg{I.rec, I.h, I.w, I.label0 + I.fw};
        }
    }
    cs->label_total = label_total;
    if (label_total) DECODE_CK(cs->labels.grow((size_t)label_total));
    if (view3d) DECODE_CK(cs->segs.grow((size_t)n * PANEL_ELEMS));
    return 0;
}

}  // namespace smapb
