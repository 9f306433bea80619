// Huffman JPEG decoding on the GPU (jpeg.cu): host marker walk + batched device phases.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

namespace smapb {

struct JpegWorkspace;  // handle-owned device / pinned buffers, grown on demand

JpegWorkspace* jpeg_workspace_create();
void jpeg_workspace_destroy(JpegWorkspace* ws);

// Decodes the images whose headers the decoder accepts into bgr[i] (uint8 [out_h, out_w, 3], device), and reports
// status[i] (SMAPB_JPEG_*) for every image.  flags = 0 accepts baseline files only; SMAPB_JPEG_SCANS also accepts
// sequential files with several scans and progressive Huffman files; SMAPB_JPEG_COLOUR also accepts CMYK, YCCK and
// RGB frames and every integral sampling, in either mode.  The scans run in rounds, the r-th scan of every
// image in round r.  Synchronises `st` before returning.  0 on success; otherwise a CUDA error or -1 for bad arguments,
// with the text in *err.  *launches is incremented by the number of kernels launched.
int jpeg_decode(JpegWorkspace* ws, int n, const uint8_t* const* jpeg, const int64_t* nbytes, uint8_t* const* bgr, int flags,
                int* status, cudaStream_t st, int64_t* launches, std::string* err);

}  // namespace smapb
