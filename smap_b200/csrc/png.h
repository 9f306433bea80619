// PNG decoding on the GPU (png.cu): host chunk walk + batched device phases with a block-parallel inflate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

namespace smapb {

struct PngWorkspace;  // handle-owned device / pinned buffers, grown on demand

PngWorkspace* png_workspace_create();
void png_workspace_destroy(PngWorkspace* ws);

// Decodes the files whose chunk walk png.cu accepts into bgr[i] (uint8 [out_h, out_w, 3], device), and reports status[i]
// (SMAPB_JPEG_*) for every file.  Synchronises `st` before returning.  0 on success; otherwise a CUDA error or -1 for bad
// arguments, with the text in *err.  *launches is incremented by the number of kernels launched.
int png_decode(PngWorkspace* ws, int n, const uint8_t* const* png, const int64_t* nbytes, uint8_t* const* bgr, int* status,
               cudaStream_t st, int64_t* launches, std::string* err);

// The last png_decode's inflate counters: candidates the block finder listed, those the chain did not start a block at
// (false positives), chained blocks confirmed through the finder, chained blocks the serial walk handled itself.
void png_last_stats(const PngWorkspace* ws, int64_t out[4]);

}  // namespace smapb
