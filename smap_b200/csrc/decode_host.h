// Host pieces the JPEG and PNG batch drivers share (jpeg.cu, png.cu): buffer growth, the CUDA check, the buffers both
// workspaces hold, the start of a batch decode and the report of the header-only info entry points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/smap_b200.h"

// Returns -10 from the enclosing function, with the call, CUDA's error text and the source position in *err.
#define DECODE_CK(call)                                                                                          \
    do {                                                                                                         \
        cudaError_t e_ = (call);                                                                                 \
        if (e_ != cudaSuccess) {                                                                                 \
            *err = std::string(#call) + ": " + cudaGetErrorString(e_) + " @" + __FILE_NAME__ + ":" +              \
                   std::to_string(__LINE__);                                                                     \
            return -10;                                                                                          \
        }                                                                                                        \
    } while (0)

namespace smapb {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Makes *p hold at least n elements, device memory or pinned host memory; a buffer that grows loses its contents.
template <typename T>
cudaError_t grow_buffer(T** p, size_t* cap, size_t n, bool pinned) {
    if (n <= *cap) return cudaSuccess;
    if (*p) pinned ? cudaFreeHost(*p) : cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    cudaError_t e = pinned ? cudaMallocHost((void**)p, n * sizeof(T)) : cudaMalloc((void**)p, n * sizeof(T));
    if (e == cudaSuccess) *cap = n;
    return e;
}

template <typename T>
cudaError_t grow(T** p, size_t* cap, size_t n) { return grow_buffer(p, cap, n, false); }

template <typename T>
cudaError_t grow_pinned(T** p, size_t* cap, size_t n) { return grow_buffer(p, cap, n, true); }

// The buffers of both workspaces: the pinned staging area of a batch (descriptors and file bytes, one upload per batch),
// its device copy, a small device area (statuses and counters, laid out by each driver) and its pinned mirror.
struct DecodeBuffers {
    uint8_t* host = nullptr;
    size_t host_cap = 0;
    uint8_t* dev_in = nullptr;
    size_t dev_in_cap = 0;
    int* small = nullptr;
    size_t small_cap = 0;
    int* small_host = nullptr;
    size_t small_host_cap = 0;
};

inline void free_decode_buffers(DecodeBuffers* b) {
    if (b->host) cudaFreeHost(b->host);
    if (b->small_host) cudaFreeHost(b->small_host);
    if (b->dev_in) cudaFree(b->dev_in);
    if (b->small) cudaFree(b->small);
}

// The start of a batch decode.  Checks the arguments, refuses a stream under capture (the drivers synchronise and may
// grow their workspaces), walks every file's header into (*H)[i] and status[i] with walk(data, nbytes, &header), and
// requires an output buffer for every file the walk accepts.  Returns the number of accepted files, listed in *idx, or
// the driver's error code with the text, prefixed by name, in *err.
template <typename Header, typename Walk>
int decode_preamble(const char* name, int n, const uint8_t* const* data, const int64_t* nbytes, uint8_t* const* out,
                    int* status, cudaStream_t st, Walk walk, std::vector<Header>* H, std::vector<int>* idx, std::string* err) {
    if (n < 0 || (n > 0 && (!data || !nbytes || !out || !status))) {
        *err = std::string(name) + ": null argument";
        return -1;
    }
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    DECODE_CK(cudaStreamIsCapturing(st, &cap));
    if (cap != cudaStreamCaptureStatusNone) {
        *err = std::string(name) + ": not capturable (it synchronises and may grow its workspace)";
        return -1;
    }
    H->resize(n);
    for (int i = 0; i < n; i++) {
        status[i] = walk(data[i], nbytes[i], &(*H)[i]);
        if (status[i] == SMAPB_JPEG_OK) {
            if (!out[i]) {
                *err = std::string(name) + ": no output buffer for decodable image " + std::to_string(i);
                return -1;
            }
            idx->push_back(i);
        }
    }
    return (int)idx->size();
}

// What the header-only info entry points report for a walk's status and header: the output size and orientation of an
// accepted file, zeros otherwise.
template <typename Header>
int report_info(int walk_status, const Header& H, int* status, int* h, int* w, int* orientation) {
    *status = walk_status;
    const bool ok = walk_status == SMAPB_JPEG_OK;
    if (h) *h = ok ? H.out_h : 0;
    if (w) *w = ok ? H.out_w : 0;
    if (orientation) *orientation = ok ? H.orientation : 0;
    return 0;
}

}  // namespace smapb
