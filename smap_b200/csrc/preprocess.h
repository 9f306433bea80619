// Inference pre-processing (SURVEY.md 8(f) f1): dataset/custom_dataset.py:27-68 (cv2.resize INTER_LINEAR on uint8 BGR,
// gray-128 letterbox, torchvision ToTensor + Normalize) as one kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace smapb {

// resampling plan of one source geometry, host side (uploaded once per geometry and cached by the handle)
struct ResizePlan {
    int src_w = 0, src_h = 0, dst_w = 0, dst_h = 0;  // dst = cvRound(src * scale)
    int pad_l = 0, pad_t = 0;                        // letterbox offsets inside the net input
    int mode = 0;                                    // 0 bilinear (fixed point), 1 exact 1/2 scale (2x2 rounded mean), 2 copy
    double scale = 1.0;                              // min(net_w / src_w, net_h / src_h)
    std::vector<int> xofs, yofs;                     // [dst_w] left tap; [dst_h][2] clamped rows
    std::vector<short> xcoef, ycoef;                 // [dst_w][2], [dst_h][2]  (weights * 2048, rounded half to even)
};

// fills `plan` for a src_w x src_h image going into a net_w x net_h input; false (plan unusable) for sides outside
// [1, 16384] and where cv2.resize refuses the image: a resized side that rounds to 0 pixels
bool make_resize_plan(int src_w, int src_h, int net_w, int net_h, ResizePlan* plan);

struct ResizeTablesDev {
    const int* xofs;
    const short* xcoef;
    const int* yofs;
    const short* ycoef;
};

// bgr: uint8 [src_h, src_w, 3] (device), out: fp32 [3, net_h, net_w] (device)
cudaError_t launch_preprocess(const uint8_t* bgr, const ResizePlan& plan, const ResizeTablesDev& tab, int net_w, int net_h,
                              float* out, cudaStream_t st);

}  // namespace smapb
