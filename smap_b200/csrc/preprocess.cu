// uint8 BGR HWC image -> letterboxed, normalised fp32 NCHW network input, bit-identical to the reference's
// cv2.resize(img, (0,0), fx=s, fy=s) + gray-128 padding + ToTensor + Normalize (dataset/custom_dataset.py:23-24,42-68).
//
// cv2's 8-bit bilinear resize is fixed point (OpenCV modules/imgproc/src/resize.cpp): float32 weights rounded (half to
// even) to multiples of 1/2048, 32-bit horizontal sums, vertical pass
//   (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2
// and an exact 1/2 scale is rerouted to INTER_AREA (rounded mean of 2x2 blocks, or of the pixels inside a block cut by an
// odd last column or row).  The tables are built on the host with the
// same float/double operations (make_resize_plan); the kernel does the integer arithmetic and the normalisation with
// IEEE division, one thread per output pixel (3 channels), fully coalesced fp32 stores.  HBM-bound: reads the source
// image once (through L1/L2, each source pixel is touched by <= 2x2 output pixels when down-scaling), writes 5.1 MB.
#include "preprocess.h"

#include <math.h>

namespace smapb {

static inline int cv_round(double v) { return (int)lrint(v); }  // round half to even (default rounding mode)

bool make_resize_plan(int src_w, int src_h, int net_w, int net_h, ResizePlan* P) {
    if (src_w < 1 || src_h < 1 || src_w > 16384 || src_h > 16384 || net_w < 1 || net_h < 1) return false;
    P->src_w = src_w;
    P->src_h = src_h;
    const double s = fmin((double)net_w / src_w, (double)net_h / src_h);  // custom_dataset.py:46
    P->scale = s;
    P->dst_w = cv_round(src_w * s);  // cv::resize: dsize = Size(saturate_cast<int>(ssize.width * fx), ...)
    P->dst_h = cv_round(src_h * s);
    if (P->dst_w == 0 || P->dst_h == 0) return false;  // cv::resize asserts !dsize.empty(): e.g. 16x16384 -> rint(0.5) = 0
    P->pad_l = P->pad_t = 0;
    if (P->dst_w < net_w) P->pad_l = (net_w - P->dst_w) / 2;       // custom_dataset.py:55-60
    else if (P->dst_h < net_h) P->pad_t = (net_h - P->dst_h) / 2;  // custom_dataset.py:61-66
    const double inv = 1.0 / s;
    if (P->dst_w == src_w && P->dst_h == src_h) {
        P->mode = 2;
    } else if ((int)inv == 2 && fabs(2.0 - inv) < 2.220446049250313e-16) {
        P->mode = 1;
    } else {
        P->mode = 0;
    }
    P->xofs.assign(P->dst_w, 0);
    P->xcoef.assign((size_t)P->dst_w * 2, 0);
    P->yofs.assign((size_t)P->dst_h * 2, 0);
    P->ycoef.assign((size_t)P->dst_h * 2, 0);
    if (P->mode != 0) return true;
    for (int d = 0; d < P->dst_w; d++) {
        float f = (float)((d + 0.5) * inv - 0.5);
        int sx = (int)floorf(f);
        f -= (float)sx;
        if (sx < 0) f = 0.f, sx = 0;
        if (sx >= src_w - 1) f = 0.f, sx = src_w - 1;
        P->xofs[d] = sx;
        P->xcoef[2 * d] = (short)lrintf((1.f - f) * 2048.f);
        P->xcoef[2 * d + 1] = (short)lrintf(f * 2048.f);
    }
    for (int d = 0; d < P->dst_h; d++) {
        float f = (float)((d + 0.5) * inv - 0.5);
        const int sy = (int)floorf(f);
        f -= (float)sy;
        P->yofs[2 * d] = sy < 0 ? 0 : (sy > src_h - 1 ? src_h - 1 : sy);              // rows are clamped, weights are not snapped
        P->yofs[2 * d + 1] = sy + 1 < 0 ? 0 : (sy + 1 > src_h - 1 ? src_h - 1 : sy + 1);
        P->ycoef[2 * d] = (short)lrintf((1.f - f) * 2048.f);
        P->ycoef[2 * d + 1] = (short)lrintf(f * 2048.f);
    }
    return true;
}

__global__ void __launch_bounds__(256) preprocess_kernel(const uint8_t* __restrict__ src, int src_w, int src_h, int dst_w,
                                                         int dst_h, int pad_l, int pad_t, int mode, ResizeTablesDev tab, int net_w,
                                                         int net_h, float* __restrict__ out) {
    const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
    if (x >= net_w || y >= net_h) return;
    const int dx = x - pad_l, dy = y - pad_t;
    int v[3] = {128, 128, 128};  // letterbox gray
    if (dx >= 0 && dx < dst_w && dy >= 0 && dy < dst_h) {
        if (mode == 2) {
            const uint8_t* p = src + ((size_t)dy * src_w + dx) * 3;
            v[0] = p[0], v[1] = p[1], v[2] = p[2];
        } else if (mode == 1) {
            const int nx = min(2, src_w - 2 * dx), ny = min(2, src_h - 2 * dy);  // 1 where rint(src / 2) rounded up
            const uint8_t* p = src + ((size_t)(2 * dy) * src_w + 2 * dx) * 3;
            const uint8_t* q = p + (size_t)src_w * 3;
            if (nx == 2 && ny == 2) {
#pragma unroll
                for (int c = 0; c < 3; c++) v[c] = ((int)p[c] + (int)p[3 + c] + (int)q[c] + (int)q[3 + c] + 2) >> 2;
            } else {  // window cut by the last column / row: cv2's saturate_cast<uchar>((float)sum / count), half to even
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    int sum = p[c];
                    if (nx == 2) sum += p[3 + c];
                    if (ny == 2) sum += q[c];
                    v[c] = __float2int_rn(__fdiv_rn((float)sum, (float)(nx * ny)));
                }
            }
        } else {
            const int sx = tab.xofs[dx];
            const int sx1 = min(sx + 1, src_w - 1);
            const int a0 = tab.xcoef[2 * dx], a1 = tab.xcoef[2 * dx + 1];
            const int y0 = tab.yofs[2 * dy], y1 = tab.yofs[2 * dy + 1];
            const int b0 = tab.ycoef[2 * dy], b1 = tab.ycoef[2 * dy + 1];
            const uint8_t* r0 = src + (size_t)y0 * src_w * 3;
            const uint8_t* r1 = src + (size_t)y1 * src_w * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const int h0 = (int)r0[sx * 3 + c] * a0 + (int)r0[sx1 * 3 + c] * a1;  // HResizeLinear: 32-bit sums (x 2048)
                const int h1 = (int)r1[sx * 3 + c] * a0 + (int)r1[sx1 * 3 + c] * a1;
                int o = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;  // VResizeLinear<uchar,int,short,FixedPtCast<..,22>>
                v[c] = o < 0 ? 0 : (o > 255 ? 255 : o);
            }
        }
    }
    // ToTensor: float32(u8) / 255; Normalize: (x - mean) / std, BGR means/stds of exps/stage3_root2/config.py:34-35
    const float mean[3] = {0.406f, 0.456f, 0.485f}, stdv[3] = {0.225f, 0.224f, 0.229f};
    const size_t plane = (size_t)net_w * net_h;
#pragma unroll
    for (int c = 0; c < 3; c++)
        out[c * plane + (size_t)y * net_w + x] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v[c], 255.f), mean[c]), stdv[c]);
}

cudaError_t launch_preprocess(const uint8_t* bgr, const ResizePlan& P, const ResizeTablesDev& tab, int net_w, int net_h, float* out,
                              cudaStream_t st) {
    dim3 block(32, 8), grid((net_w + 31) / 32, (net_h + 7) / 8);
    preprocess_kernel<<<grid, block, 0, st>>>(bgr, P.src_w, P.src_h, P.dst_w, P.dst_h, P.pad_l, P.pad_t, P.mode, tab, net_w, net_h, out);
    return cudaGetLastError();
}

}  // namespace smapb
