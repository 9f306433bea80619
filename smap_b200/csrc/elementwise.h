// Launch interface of the non-GEMM backbone kernels (elementwise.cu).
// Activations are NHWC "split-bf16": plane 0 = hi, plane 1 (at + plane_stride elements) = lo; terms = 1 or 2 planes.
// f16 = true: one plane of fp16 elements instead (the pointers are 2-byte storage either way); kernels that compute new
// values clamp them to +-65504 and add the number of clamped elements to *sat.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace smapb {
cudaError_t launch_f32_to_split(const float* x, __nv_bfloat16* out, long long n, long long plane_stride, int terms,
                                cudaStream_t st, bool f16 = false);
cudaError_t launch_stem(const float* x_nchw, const float* wgt, const float* bias, int N, int H, int W,
                        __nv_bfloat16* out, long long plane_stride, int terms, cudaStream_t st, bool f16 = false,
                        unsigned long long* sat = nullptr);
cudaError_t launch_s2d(const float* x_nchw, int N, int H, int W, __nv_bfloat16* out, long long plane_stride, int terms,
                       cudaStream_t st, bool f16 = false, unsigned long long* sat = nullptr);
cudaError_t launch_maxpool(const __nv_bfloat16* in, long long in_ps, int N, int H, int W, int C, __nv_bfloat16* out,
                           long long out_ps, int terms, cudaStream_t st, bool f16 = false);
cudaError_t launch_upadd_relu(const __nv_bfloat16* a, long long a_ps, const __nv_bfloat16* t, long long t_ps, int N,
                              int H, int W, int Hi, int Wi, int C, __nv_bfloat16* out, long long out_ps, int terms,
                              cudaStream_t st, bool f16 = false, unsigned long long* sat = nullptr);
cudaError_t launch_head_merge(const float* r4, const float* r3, const float* r2, int N, int H, int W, int H3, int W3,
                              int H2, int W2, int Cpad, int Cout, float* out, cudaStream_t st);
cudaError_t launch_tapsum(const float* T, const float* bias, int N, int H, int W, int Cpad, int C, float* out,
                          cudaStream_t st);
cudaError_t launch_merge_scale(float* hm, const float* hm_flip, int B, int h, int w, int do_scale, cudaStream_t st);
}  // namespace smapb
