// Non-GEMM kernels of the backbone (HBM-bound, NHWC split-bf16 or fp16 activations): stem 7x7 conv, max-pool,
// bilinear(align_corners) up-sample + add + ReLU, head merge + NHWC->NCHW, flip-TTA merge / rescale.
// Kernels that write activations are templated on the element format E (common.cuh).  The fp16 variants clamp every value
// they compute to +-65504 and add the number of clamped elements to the handle's saturation counter.
#include "elementwise.h"
#include "common.cuh"

namespace smapb {

// ---------------------------------------------------------------------------------------------
// fp32 NHWC -> split-bf16 planes (test hook + generic converter)
// ---------------------------------------------------------------------------------------------
template <class E>
__global__ void f32_to_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, long long n,
                                    long long plane_stride, int terms) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if constexpr (E::F16) {
        reinterpret_cast<__half*>(out)[i] = __float2half_rn(x[i]);
    } else {
        __nv_bfloat16 h, l;
        split_bf16(x[i], h, l);
        out[i] = h;
        if (terms == 2) out[plane_stride + i] = l;
    }
}
cudaError_t launch_f32_to_split(const float* x, __nv_bfloat16* out, long long n, long long plane_stride, int terms,
                                cudaStream_t st, bool f16) {
    if (f16)
        f32_to_split_kernel<ElemF16><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, out, n, plane_stride, terms);
    else
        f32_to_split_kernel<ElemBF16><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, out, n, plane_stride, terms);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Stem: conv 7x7 stride 2 pad 3, 3 -> 64, folded BN + ReLU (model/smap.py:83-85), fp32 FFMA.
// Input fp32 NCHW [N,3,H,W]; output split-bf16 NHWC [N,H/2,W/2,64].
// CTA = 8 x 32 output pixels x 64 channels; thread = one pixel, 4 passes of 16 channels.
// ---------------------------------------------------------------------------------------------
constexpr int ST_TW = 128, ST_TH = 8;                         // output tile per CTA
constexpr int ST_PX = 4;                                        // adjacent output pixels per thread
constexpr int ST_PW = ST_TW * 2 + 5, ST_PH = ST_TH * 2 + 5;     // input patch 261 x 21
constexpr int ST_PWP = ST_PW + 3;                               // padded row pitch

// thread = 4 adjacent output pixels x 16 channels (4 passes over the channel groups): per (ky, ci) row the 13 input
// values and the 7x16 weights are loaded once and feed 448 FFMAs (11 FFMA per shared-memory load).
template <class E>
__global__ void __launch_bounds__(256, 2)
stem_kernel(const float* __restrict__ x, const float* __restrict__ wgt /*[147][64] (ky,kx,ci) x co*/,
            const float* __restrict__ bias, int H, int W, __nv_bfloat16* __restrict__ out, long long plane_stride,
            int terms, unsigned long long* sat) {
    extern __shared__ __align__(16) float stem_smem[];
    float* s_w = stem_smem;                   // [147*64]
    float* s_in = stem_smem + 147 * 64;       // [3][ST_PH][ST_PWP]
    const int Ho = H / 2, Wo = W / 2;
    const int n = blockIdx.z;
    const int oy0 = blockIdx.y * ST_TH, ox0 = blockIdx.x * ST_TW;
    const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
    for (int i = threadIdx.x; i < 147 * 64; i += 256) s_w[i] = wgt[i];
    for (int i = threadIdx.x; i < 3 * ST_PH * ST_PW; i += 256) {
        const int c = i / (ST_PH * ST_PW), r = i - c * (ST_PH * ST_PW);
        const int py = r / ST_PW, px = r - py * ST_PW;
        const int iy = iy0 + py, ix = ix0 + px;
        float v = 0.f;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)n * 3 + c) * H + iy) * W + ix];
        s_in[(c * ST_PH + py) * ST_PWP + px] = v;
    }
    __syncthreads();
    const int ty = threadIdx.x / (ST_TW / ST_PX), tx = (threadIdx.x % (ST_TW / ST_PX)) * ST_PX;
    const int oy = oy0 + ty;
    int n_sat = 0;
#pragma unroll 1
    for (int cg = 0; cg < 4; cg++) {
        float acc[ST_PX][16];
#pragma unroll
        for (int p = 0; p < ST_PX; p++)
#pragma unroll
            for (int j = 0; j < 16; j++) acc[p][j] = 0.f;
#pragma unroll 1
        for (int ky = 0; ky < 7; ky++) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                float in[16];  // 13 used; 4 x LDS.128 (row pitch and tx*2 keep 16-byte alignment)
                const float4* row4 = reinterpret_cast<const float4*>(s_in + (c * ST_PH + ty * 2 + ky) * ST_PWP + tx * 2);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const float4 q = row4[i];
                    in[4 * i] = q.x, in[4 * i + 1] = q.y, in[4 * i + 2] = q.z, in[4 * i + 3] = q.w;
                }
#pragma unroll
                for (int kx = 0; kx < 7; kx++) {
                    const float4* wp = reinterpret_cast<const float4*>(&s_w[((ky * 7 + kx) * 3 + c) * 64 + cg * 16]);
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const float4 w4 = wp[j];
#pragma unroll
                        for (int p = 0; p < ST_PX; p++) {
                            const float v = in[2 * p + kx];
                            acc[p][4 * j + 0] = fmaf(v, w4.x, acc[p][4 * j + 0]);
                            acc[p][4 * j + 1] = fmaf(v, w4.y, acc[p][4 * j + 1]);
                            acc[p][4 * j + 2] = fmaf(v, w4.z, acc[p][4 * j + 2]);
                            acc[p][4 * j + 3] = fmaf(v, w4.w, acc[p][4 * j + 3]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int p = 0; p < ST_PX; p++) {
            const int ox = ox0 + tx + p;
            if (oy < Ho && ox < Wo) {
                const size_t obase = (((size_t)n * Ho + oy) * Wo + ox) * 64;
                uint32_t hw_[8], lw_[8];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float a = fmaxf(acc[p][2 * j] + bias[cg * 16 + 2 * j], 0.f);
                    const float b = fmaxf(acc[p][2 * j + 1] + bias[cg * 16 + 2 * j + 1], 0.f);
                    if constexpr (E::F16) {
                        hw_[j] = E::pack2(E::clamp(a, n_sat), E::clamp(b, n_sat));
                    } else {
                        __nv_bfloat16 ah, al, bh, bl;
                        split_bf16(a, ah, al);
                        split_bf16(b, bh, bl);
                        hw_[j] = pack_bf16x2(ah, bh);
                        lw_[j] = pack_bf16x2(al, bl);
                    }
                }
                uint4* oh = reinterpret_cast<uint4*>(out + obase + cg * 16);
                oh[0] = make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]);
                oh[1] = make_uint4(hw_[4], hw_[5], hw_[6], hw_[7]);
                if constexpr (!E::F16) {
                    if (terms == 2) {
                        uint4* ol = reinterpret_cast<uint4*>(out + plane_stride + obase + cg * 16);
                        ol[0] = make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]);
                        ol[1] = make_uint4(lw_[4], lw_[5], lw_[6], lw_[7]);
                    }
                }
            }
        }
    }
    if constexpr (E::F16) saturation_add(sat, n_sat);
}
template <class E>
cudaError_t launch_stem_e(const float* x, const float* wgt, const float* bias, int N, int H, int W, __nv_bfloat16* out,
                          long long plane_stride, int terms, cudaStream_t st, unsigned long long* sat) {
    const int Ho = H / 2, Wo = W / 2;
    dim3 grid((Wo + ST_TW - 1) / ST_TW, (Ho + ST_TH - 1) / ST_TH, N);
    constexpr int smem = (147 * 64 + 3 * ST_PH * ST_PWP) * 4;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(stem_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    stem_kernel<E><<<grid, 256, smem, st>>>(x, wgt, bias, H, W, out, plane_stride, terms, sat);
    return cudaGetLastError();
}
cudaError_t launch_stem(const float* x, const float* wgt, const float* bias, int N, int H, int W, __nv_bfloat16* out,
                        long long plane_stride, int terms, cudaStream_t st, bool f16, unsigned long long* sat) {
    return f16 ? launch_stem_e<ElemF16>(x, wgt, bias, N, H, W, out, plane_stride, terms, st, sat)
               : launch_stem_e<ElemBF16>(x, wgt, bias, N, H, W, out, plane_stride, terms, st, sat);
}

// ---------------------------------------------------------------------------------------------
// Space-to-depth of the network input for the tensor-core stem: fp32 NCHW [N,3,H,W] ->
// split-bf16 [plane][N][H/2][W/2 + 3][16] with channel (by*2+bx)*3 + c = in[c][2y+by][2x+bx] (12 used, 4 zero) and
// zero pixel columns 0,1 (left) and W/2+2 (right), so that every 4-pixel sliding window [x-2, x+1] of the 7x7/s2
// receptive field is a contiguous, in-bounds 128-byte row for TMA.
// ---------------------------------------------------------------------------------------------
template <class E>
__global__ void s2d_kernel(const float* __restrict__ x, int N, int H, int W, __nv_bfloat16* __restrict__ out,
                           long long plane_stride, int terms, unsigned long long* sat) {
    const int H2 = H / 2, W2 = W / 2, WP = W2 + 3;
    const long long total = (long long)N * H2 * WP;
    int n_sat = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xp = (int)(i % WP);
        long long r = i / WP;
        const int y2 = (int)(r % H2);
        const int n = (int)(r / H2);
        const int x2 = xp - 2;
        float v[16];
#pragma unroll
        for (int j = 0; j < 16; j++) v[j] = 0.f;
        if (x2 >= 0 && x2 < W2) {
#pragma unroll
            for (int c = 0; c < 3; c++)
#pragma unroll
                for (int by = 0; by < 2; by++) {
                    const float2 p2 = *reinterpret_cast<const float2*>(x + (((size_t)n * 3 + c) * H + 2 * y2 + by) * W + 2 * x2);
                    v[(by * 2 + 0) * 3 + c] = p2.x;
                    v[(by * 2 + 1) * 3 + c] = p2.y;
                }
        }
        uint32_t hw_[8], lw_[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if constexpr (E::F16) {
                hw_[j] = E::pack2(E::clamp(v[2 * j], n_sat), E::clamp(v[2 * j + 1], n_sat));
            } else {
                __nv_bfloat16 ah, al, bh, bl;
                split_bf16(v[2 * j], ah, al);
                split_bf16(v[2 * j + 1], bh, bl);
                hw_[j] = pack_bf16x2(ah, bh);
                lw_[j] = pack_bf16x2(al, bl);
            }
        }
        uint4* oh = reinterpret_cast<uint4*>(out + i * 16);
        oh[0] = make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]);
        oh[1] = make_uint4(hw_[4], hw_[5], hw_[6], hw_[7]);
        if constexpr (!E::F16) {
            if (terms == 2) {
                uint4* ol = reinterpret_cast<uint4*>(out + plane_stride + i * 16);
                ol[0] = make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]);
                ol[1] = make_uint4(lw_[4], lw_[5], lw_[6], lw_[7]);
            }
        }
    }
    if constexpr (E::F16) saturation_add(sat, n_sat);
}
cudaError_t launch_s2d(const float* x, int N, int H, int W, __nv_bfloat16* out, long long plane_stride, int terms,
                       cudaStream_t st, bool f16, unsigned long long* sat) {
    const long long total = (long long)N * (H / 2) * (W / 2 + 3);
    const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    if (f16)
        s2d_kernel<ElemF16><<<blocks, 256, 0, st>>>(x, N, H, W, out, plane_stride, terms, sat);
    else
        s2d_kernel<ElemBF16><<<blocks, 256, 0, st>>>(x, N, H, W, out, plane_stride, terms, sat);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// helpers on 8-channel packets (uint4 = 8 bf16)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void unpack8(const uint4& h, const uint4& l, float (&v)[8]) {
    const uint32_t hh[4] = {h.x, h.y, h.z, h.w}, ll[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 4; e++) {
        v[2 * e] = bf16lo_to_f(hh[e]) + bf16lo_to_f(ll[e]);
        v[2 * e + 1] = bf16hi_to_f(hh[e]) + bf16hi_to_f(ll[e]);
    }
}
__device__ __forceinline__ void pack8(const float (&v)[8], uint4& h, uint4& l) {
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int e = 0; e < 4; e++) {
        __nv_bfloat16 a, b, c, d;
        split_bf16(v[2 * e], a, b);
        split_bf16(v[2 * e + 1], c, d);
        hh[e] = pack_bf16x2(a, c);
        ll[e] = pack_bf16x2(b, d);
    }
    h = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    l = make_uint4(ll[0], ll[1], ll[2], ll[3]);
}
template <class E>
__device__ __forceinline__ void load8(const __nv_bfloat16* p, long long plane_stride, int terms, float (&v)[8]) {
    const uint4 h = *reinterpret_cast<const uint4*>(p);
    if constexpr (E::F16) {
        const uint32_t hh[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
        for (int e = 0; e < 4; e++) v[2 * e] = E::lo(hh[e]), v[2 * e + 1] = E::hi(hh[e]);
    } else {
        const uint4 l = (terms == 2) ? *reinterpret_cast<const uint4*>(p + plane_stride) : make_uint4(0, 0, 0, 0);
        unpack8(h, l, v);
    }
}
// fp16: values outside +-65504 are clamped and counted in n_sat
template <class E>
__device__ __forceinline__ void store8(__nv_bfloat16* p, long long plane_stride, int terms, const float (&v)[8], int& n_sat) {
    if constexpr (E::F16) {
        *reinterpret_cast<uint4*>(p) = make_uint4(E::pack2(E::clamp(v[0], n_sat), E::clamp(v[1], n_sat)),
                                                  E::pack2(E::clamp(v[2], n_sat), E::clamp(v[3], n_sat)),
                                                  E::pack2(E::clamp(v[4], n_sat), E::clamp(v[5], n_sat)),
                                                  E::pack2(E::clamp(v[6], n_sat), E::clamp(v[7], n_sat)));
    } else {
        uint4 h, l;
        pack8(v, h, l);
        *reinterpret_cast<uint4*>(p) = h;
        if (terms == 2) *reinterpret_cast<uint4*>(p + plane_stride) = l;
    }
}

// ---------------------------------------------------------------------------------------------
// MaxPool 3x3 stride 2 pad 1 (model/smap.py:86).  Input is post-ReLU (>= 0) so zero padding == -inf padding.
// ---------------------------------------------------------------------------------------------
template <class E>
__global__ void maxpool_kernel(const __nv_bfloat16* __restrict__ in, long long in_ps, int N, int H, int W, int C,
                               __nv_bfloat16* __restrict__ out, long long out_ps, int terms) {
    int n_sat = 0;  // the maximum of stored values is a stored value: nothing to clamp
    const int Ho = H / 2, Wo = W / 2, CG = C / 8;
    const long long total = (long long)N * Ho * Wo * CG;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(i % CG);
        long long r = i / CG;
        const int ox = (int)(r % Wo);
        r /= Wo;
        const int oy = (int)(r % Ho);
        const int n = (int)(r / Ho);
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; j++) m[j] = 0.f;
        for (int dy = -1; dy <= 1; dy++) {
            const int iy = oy * 2 + dy;
            if (iy < 0 || iy >= H) continue;
            for (int dx = -1; dx <= 1; dx++) {
                const int ix = ox * 2 + dx;
                if (ix < 0 || ix >= W) continue;
                float v[8];
                load8<E>(in + (((long long)n * H + iy) * W + ix) * C + cg * 8, in_ps, terms, v);
#pragma unroll
                for (int j = 0; j < 8; j++) m[j] = fmaxf(m[j], v[j]);
            }
        }
        store8<E>(out + (((long long)n * Ho + oy) * Wo + ox) * C + cg * 8, out_ps, terms, m, n_sat);
    }
}
cudaError_t launch_maxpool(const __nv_bfloat16* in, long long in_ps, int N, int H, int W, int C, __nv_bfloat16* out,
                           long long out_ps, int terms, cudaStream_t st, bool f16) {
    const long long total = (long long)N * (H / 2) * (W / 2) * (C / 8);
    const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    if (f16)
        maxpool_kernel<ElemF16><<<blocks, 256, 0, st>>>(in, in_ps, N, H, W, C, out, out_ps, terms);
    else
        maxpool_kernel<ElemBF16><<<blocks, 256, 0, st>>>(in, in_ps, N, H, W, C, out, out_ps, terms);
    return cudaGetLastError();
}

// bilinear source taps and weights of output index o, align_corners=True
__device__ __forceinline__ void bilin_coeff(int o, int in, int out, int& i0, int& i1, float& l0, float& l1) {
    // ATen area_pixel_compute_source_index with align_corners: src = o * (in-1)/(out-1)
    const float scale = (out > 1) ? (float)(in - 1) / (float)(out - 1) : 0.f;
    const float src = scale * (float)o;
    i0 = (int)src;
    i1 = i0 + ((i0 < in - 1) ? 1 : 0);
    l1 = src - (float)i0;
    l0 = 1.f - l1;
}

// ---------------------------------------------------------------------------------------------
// Head merge: out[n,c,y,x] = (r4 + up(r3)) + up(r2) (model/smap.py:418 with :221) and NHWC(fp32, padded C)
// -> NCHW fp32.  r3 / r2 may be null (plain transpose for det_d / root_d).  CTA = 32 pixels of one row.
// ---------------------------------------------------------------------------------------------
// bilinear tap combination in the contraction pattern the scalar expression
//   h0 * (w0 * b00 + w1 * b01) + h1 * (w0 * b10 + w1 * b11)
// compiled to in the scalar form of this kernel (PTX of the round-1/2 builds: the row sums fuse their SECOND product,
// the column sum its FIRST), pinned so that the result does not depend on how the surrounding code is written
__device__ __forceinline__ float bilin4(float h0, float h1, float w0, float w1, float b00, float b01, float b10, float b11) {
    const float s0 = __fmaf_rn(w1, b01, __fmul_rn(w0, b00));
    const float s1 = __fmaf_rn(w1, b11, __fmul_rn(w0, b10));
    return __fmaf_rn(h0, s0, __fmul_rn(h1, s1));
}

// One thread = 4 channels (one 16-byte load per tap) of one pixel; the x coefficients of the CTA's 32 pixels are computed
// once.  Channel groups above Cout are never read.
__global__ void __launch_bounds__(256)
head_merge_kernel(const float* __restrict__ r4, const float* __restrict__ r3, const float* __restrict__ r2, int N, int H,
                  int W, int H3, int W3, int H2, int W2, int Cpad, int Cout, float* __restrict__ out) {
    __shared__ float tile[64][33];
    __shared__ int s_xi[32][4];    // xa0, xa1, xb0, xb1
    __shared__ float s_xw[32][4];  // wa0, wa1, wb0, wb1
    const int x0 = blockIdx.x * 32, y = blockIdx.y, n = blockIdx.z;
    int y0a = 0, y1a = 0, y0b = 0, y1b = 0;
    float ha0 = 0, ha1 = 0, hb0 = 0, hb1 = 0;
    if (r3) bilin_coeff(y, H3, H, y0a, y1a, ha0, ha1);
    if (r2) bilin_coeff(y, H2, H, y0b, y1b, hb0, hb1);
    if (threadIdx.x < 32) {
        const int x = min(x0 + (int)threadIdx.x, W - 1);
        int i0 = 0, i1 = 0;
        float l0 = 0, l1 = 0;
        if (r3) bilin_coeff(x, W3, W, i0, i1, l0, l1);
        s_xi[threadIdx.x][0] = i0, s_xi[threadIdx.x][1] = i1, s_xw[threadIdx.x][0] = l0, s_xw[threadIdx.x][1] = l1;
        i0 = i1 = 0, l0 = l1 = 0;
        if (r2) bilin_coeff(x, W2, W, i0, i1, l0, l1);
        s_xi[threadIdx.x][2] = i0, s_xi[threadIdx.x][3] = i1, s_xw[threadIdx.x][2] = l0, s_xw[threadIdx.x][3] = l1;
    }
    __syncthreads();
    const int G = (Cout + 3) / 4;  // channel groups that reach the output
    for (int i = threadIdx.x; i < 32 * G; i += 256) {
        const int px = i / G, c = (i - px * G) * 4;
        const int x = x0 + px;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (x < W) {
            v = __ldg(reinterpret_cast<const float4*>(r4 + (((size_t)n * H + y) * W + x) * Cpad + c));
            if (r3) {
                const int xa0 = s_xi[px][0], xa1 = s_xi[px][1];
                const float wa0 = s_xw[px][0], wa1 = s_xw[px][1];
                const float* b = r3 + (size_t)n * H3 * W3 * Cpad + c;
                const float4 b00 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y0a * W3 + xa0) * Cpad));
                const float4 b01 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y0a * W3 + xa1) * Cpad));
                const float4 b10 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y1a * W3 + xa0) * Cpad));
                const float4 b11 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y1a * W3 + xa1) * Cpad));
                v.x = __fadd_rn(v.x, bilin4(ha0, ha1, wa0, wa1, b00.x, b01.x, b10.x, b11.x));
                v.y = __fadd_rn(v.y, bilin4(ha0, ha1, wa0, wa1, b00.y, b01.y, b10.y, b11.y));
                v.z = __fadd_rn(v.z, bilin4(ha0, ha1, wa0, wa1, b00.z, b01.z, b10.z, b11.z));
                v.w = __fadd_rn(v.w, bilin4(ha0, ha1, wa0, wa1, b00.w, b01.w, b10.w, b11.w));
            }
            if (r2) {
                const int xb0 = s_xi[px][2], xb1 = s_xi[px][3];
                const float wb0 = s_xw[px][2], wb1 = s_xw[px][3];
                const float* b = r2 + (size_t)n * H2 * W2 * Cpad + c;
                const float4 b00 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y0b * W2 + xb0) * Cpad));
                const float4 b01 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y0b * W2 + xb1) * Cpad));
                const float4 b10 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y1b * W2 + xb0) * Cpad));
                const float4 b11 = __ldg(reinterpret_cast<const float4*>(b + ((size_t)y1b * W2 + xb1) * Cpad));
                v.x = __fadd_rn(v.x, bilin4(hb0, hb1, wb0, wb1, b00.x, b01.x, b10.x, b11.x));
                v.y = __fadd_rn(v.y, bilin4(hb0, hb1, wb0, wb1, b00.y, b01.y, b10.y, b11.y));
                v.z = __fadd_rn(v.z, bilin4(hb0, hb1, wb0, wb1, b00.z, b01.z, b10.z, b11.z));
                v.w = __fadd_rn(v.w, bilin4(hb0, hb1, wb0, wb1, b00.w, b01.w, b10.w, b11.w));
            }
        }
        tile[c][px] = v.x, tile[c + 1][px] = v.y, tile[c + 2][px] = v.z, tile[c + 3][px] = v.w;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < Cout * 32; i += 256) {
        const int c = i / 32, px = i - c * 32;
        const int x = x0 + px;
        if (x < W) out[(((size_t)n * Cout + c) * H + y) * W + x] = tile[c][px];
    }
}
cudaError_t launch_head_merge(const float* r4, const float* r3, const float* r2, int N, int H, int W, int H3, int W3,
                              int H2, int W2, int Cpad, int Cout, float* out, cudaStream_t st) {
    dim3 grid((W + 31) / 32, H, N);
    head_merge_kernel<<<grid, 256, 0, st>>>(r4, r3, r2, N, H, W, H3, W3, H2, W2, Cpad, Cout, out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Thin 3x3 heads (14- and 1-channel, model/smap.py:204-208) as tap expansion: a 1x1 GEMM produces
// T[n,y,x,tap*C+c] = sum_ci w[c,ci,tap] a[n,y,x,ci] once per pixel (the 256-channel input is read once instead of
// nine times), and this kernel gathers out[n,c,y,x] = bias[c] + sum_tap T[n, y+ky-1, x+kx-1, tap*C+c] straight into
// the NCHW fp32 result.  CTA = 32 pixels of one row, smem transpose for coalesced NCHW stores.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tapsum_kernel(const float* __restrict__ T, const float* __restrict__ bias, int N, int H, int W, int Cpad, int C,
              float* __restrict__ out) {
    __shared__ float tile[16][33];
    const int x0 = blockIdx.x * 32, y = blockIdx.y, n = blockIdx.z;
    for (int i = threadIdx.x; i < 32 * C; i += 256) {
        const int px = i / C, c = i - px * C;
        const int x = x0 + px;
        float v = 0.f;
        if (x < W) {
            v = bias[c];
#pragma unroll
            for (int ky = 0; ky < 3; ky++) {
                const int yy = y + ky - 1;
                if (yy < 0 || yy >= H) continue;
#pragma unroll
                for (int kx = 0; kx < 3; kx++) {
                    const int xx = x + kx - 1;
                    if (xx < 0 || xx >= W) continue;
                    v += T[(((size_t)n * H + yy) * W + xx) * Cpad + (ky * 3 + kx) * C + c];
                }
            }
        }
        tile[c][px] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * 32; i += 256) {
        const int c = i / 32, px = i - c * 32;
        const int x = x0 + px;
        if (x < W) out[(((size_t)n * C + c) * H + y) * W + x] = tile[c][px];
    }
}
cudaError_t launch_tapsum(const float* T, const float* bias, int N, int H, int W, int Cpad, int C, float* out,
                          cudaStream_t st) {
    if (C > 16) return cudaErrorInvalidValue;
    dim3 grid((W + 31) / 32, H, N);
    tapsum_kernel<<<grid, 256, 0, st>>>(T, bias, N, H, W, Cpad, C, out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Flip-TTA merge + per-image rescale, in place on hm [B,43,h,w] (exps/stage3_root2/test.py:55-70,111-112).
// ---------------------------------------------------------------------------------------------
__constant__ int c_flip_pair[43] = {0, 1, 2, 9, 10, 11, 12, 13, 14, 3, 4, 5, 6, 7, 8,
                                    15 + 0, 15 + 1, 15 + 2, 15 + 3, 15 + 10, 15 + 11, 15 + 12, 15 + 13, 15 + 14,
                                    15 + 15, 15 + 4, 15 + 5, 15 + 6, 15 + 7, 15 + 8, 15 + 9, 15 + 22, 15 + 23,
                                    15 + 24, 15 + 25, 15 + 26, 15 + 27, 15 + 16, 15 + 17, 15 + 18, 15 + 19, 15 + 20,
                                    15 + 21};

__global__ void merge_scale_kernel(float* __restrict__ hm, const float* __restrict__ hm_flip, int B, int h, int w,
                                   int do_scale) {
    const long long total = (long long)B * 43 * h * w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % w);
        long long r = i / w;
        const int y = (int)(r % h);
        r /= h;
        const int c = (int)(r % 43);
        const int b = (int)(r / 43);
        float v = hm[i];
        if (hm_flip) {
            const float f = hm_flip[(((long long)b * 43 + c_flip_pair[c]) * h + y) * w + (w - 1 - x)];
            if (c >= 15 && ((c - 15) & 1) == 0)
                v = __fadd_rn(v, __fmul_rn(f, -1.f));  // test.py:66
            else
                v = __fadd_rn(v, f);                    // test.py:68
            if (c >= 15) v = __fmul_rn(v, 0.5f);        // test.py:69 (key-point maps are summed, not averaged)
        }
        // test.py:111-112 `hmsIn[:15] /= 255; hmsIn[15:] /= 127` on a CUDA tensor: ATen's CUDA true-divide by a CPU
        // scalar multiplies by the fp32 reciprocal (BinaryDivTrueKernel.cu), it is not an IEEE division.
        if (do_scale) v = (c < 15) ? __fmul_rn(v, __fdiv_rn(1.f, 255.f)) : __fmul_rn(v, __fdiv_rn(1.f, 127.f));
        hm[i] = v;
    }
}
cudaError_t launch_merge_scale(float* hm, const float* hm_flip, int B, int h, int w, int do_scale, cudaStream_t st) {
    const long long total = (long long)B * 43 * h * w;
    const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    merge_scale_kernel<<<blocks, 256, 0, st>>>(hm, hm_flip, B, h, w, do_scale);
    return cudaGetLastError();
}

}  // namespace smapb
