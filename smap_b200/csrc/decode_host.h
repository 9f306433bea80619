// Host pieces the JPEG and PNG batch drivers share (jpeg.cu, png.cu), and the JPEG encoder (jpeg_enc.cu) and the
// handle (engine.h) with them: the owning device and pinned buffer, the CUDA check, the capture refusal, the start of a
// batch decode and the report of the header-only info entry points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <utility>
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

// n elements of T in device memory (cudaMalloc) or, Pinned, in page-locked host memory (cudaMallocHost), freed by the
// destructor.  Move-only; it converts to T*, so kernel launches and ConvParams take it as they take a raw pointer.
template <typename T, bool Pinned>
class Buffer {
  public:
    Buffer() = default;
    Buffer(Buffer&& o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr, o.cap_ = 0; }
    Buffer& operator=(Buffer&& o) noexcept {
        if (this != &o) {
            reset();
            std::swap(p_, o.p_);
            std::swap(cap_, o.cap_);
        }
        return *this;
    }
    ~Buffer() { reset(); }

    // Makes the buffer hold at least n elements; one that grows loses its contents.  A failed allocation leaves it empty
    // and is taken off the runtime's last-error state, so that the next launch check does not report it.
    cudaError_t grow(size_t n) {
        if (n <= cap_) return cudaSuccess;
        reset();
        void* q = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
        if (e != cudaSuccess) {
            cudaGetLastError();
            return e;
        }
        p_ = (T*)q, cap_ = n;
        return cudaSuccess;
    }
    void reset() {
        if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr, cap_ = 0;
    }
    T* get() const { return p_; }
    operator T*() const { return p_; }
    size_t capacity() const { return cap_; }

  private:
    T* p_ = nullptr;
    size_t cap_ = 0;  // elements
};
template <typename T>
using DeviceBuffer = Buffer<T, false>;
template <typename T>
using PinnedBuffer = Buffer<T, true>;

// Refuses a stream under capture: the codecs synchronise and may grow their workspaces.  0, or -1 with the text, prefixed
// by name, in *err (-10 when the stream cannot be queried).
inline int refuse_capture(const char* name, cudaStream_t st, std::string* err) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    DECODE_CK(cudaStreamIsCapturing(st, &cap));
    if (cap != cudaStreamCaptureStatusNone) {
        *err = std::string(name) + ": not capturable (it synchronises and may grow its workspace)";
        return -1;
    }
    return 0;
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
    if (int rc = refuse_capture(name, st, err)) return rc;
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
