// Baseline JPEG encoding on the GPU (jpeg_enc.cu), with an optional skeleton overlay fused into the colour pass.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/smap_b200.h"

namespace smapb {

struct JpegEncWorkspace;  // handle-owned device / pinned buffers, grown on demand

JpegEncWorkspace* jpeg_enc_workspace_create();
void jpeg_enc_workspace_destroy(JpegEncWorkspace* ws);

// Encodes n uint8 BGR frames (device) as cv2.imencode(".jpg", frame, [IMWRITE_JPEG_QUALITY, quality]) does, drawing the
// skeletons of records[i] (device, may be NULL) over frame i first; scales (device float64 [n][SMAPB_SCALE_LEN]) map their
// net-input pixels back to the frame through the letterbox of a net_w x net_h input.  flags: 0, or SMAPB_ENCODE_VIEW3D
// (records required) to encode each frame with its 3D panel on the right (view3d.cu).  The streams stay in the workspace's
// pinned buffer (jpeg_enc_result) until the next call; nbytes[i] receives their sizes.  Synchronises `st`.  0 on success;
// otherwise a CUDA error or -1 for bad arguments, with the text in *err.  *launches counts the kernels launched.
int jpeg_encode(JpegEncWorkspace* ws, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w, int quality,
                const smapb_record* records, const double* scales, int flags, int64_t* nbytes, cudaStream_t st,
                int64_t* launches, std::string* err);

// Stream i of the last jpeg_encode: its first byte, or NULL when i is out of range.
const uint8_t* jpeg_enc_result(const JpegEncWorkspace* ws, int i, int64_t* nbytes);

}  // namespace smapb
