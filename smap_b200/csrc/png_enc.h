// PNG encoding on the GPU (png_enc.cu), with the encoders' composite stage (overlay.cuh) fused into the filter pass.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/smap_b200.h"

namespace smapb {

struct PngEncWorkspace;  // handle-owned device / pinned buffers, grown on demand

PngEncWorkspace* png_enc_workspace_create();
void png_enc_workspace_destroy(PngEncWorkspace* ws);

// Encodes n uint8 BGR frames (device) as cv2.imencode(".png", frame) does, with the composite of jpeg_encode (records,
// scales and flags as there).  The files stay in the workspace's pinned buffer (png_enc_result) until the next call that
// is not refused; nbytes[i] receives their sizes.  Synchronises `st`.  0 on success; otherwise a CUDA error or -1 for bad
// arguments, with the text in *err, and the previous call's files are kept.  *launches counts the kernels launched.
int png_encode(PngEncWorkspace* ws, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
               const smapb_record* records, const double* scales, int flags, int64_t* nbytes, cudaStream_t st,
               int64_t* launches, std::string* err);

// File i of the last png_encode: its first byte, or NULL when i is out of range.
const uint8_t* png_enc_result(const PngEncWorkspace* ws, int i, int64_t* nbytes);

}  // namespace smapb
