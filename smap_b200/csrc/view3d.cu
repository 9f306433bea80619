// The 3D panel of the JPEG encoder's composite (smapb_encode_jpeg_ex with SMAPB_ENCODE_VIEW3D; rules in
// include/smap_b200.h), restated on the CPU by oracle/view3d_numpy.py.  Two launches for the whole batch:
//   setup  one CTA per image: places the joints of pred3d, reduces the fit bounds over the joints of drawn limbs, projects
//          the limbs and the 12 edges of the fit box to panel pixels, and gives each limb its paint order by a counting
//          rank (farther limbs first, ties in (row, limb) order);
//   paint  one CTA per element walks the overlay's band around it (paint.cuh) and atomicMax-es its label into the panel's
//          part of the label plane, so the painter's order comes out whatever order the CTAs run in.
// The projection is float64 with every operation rounded on its own (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn, which
// are never contracted into FMAs), so the pixels equal the oracle's.
#include <math.h>

#include "paint.cuh"
#include "view3d.h"

namespace smapb {

namespace {

constexpr int SETUP_THREADS = 512;
constexpr int NLIMB = SMAPB_MAXP * SMAPB_NL;
constexpr double kS = 0.7071067811865476;  // the float64 nearest sqrt(1/2)
constexpr double kMaxCoord = 1e15;
// the fit box's edges between corners c = (X, Y, Z) extremes selected by bits 0, 1, 2 (max when set): 4 along X, Y, Z
__constant__ int kBoxEdges[PANEL_BOX][2] = {{0, 1}, {2, 3}, {4, 5}, {6, 7}, {0, 2}, {1, 3},
                                            {4, 6}, {5, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};

__device__ __forceinline__ int persons(const smapb_record* rec) { return min(max(rec->count, 0), SMAPB_MAXP); }

// X, Y and Z finite with |.| <= 1e15 and a positive score (NaN fails every comparison)
__device__ __forceinline__ bool placed(const double* q) {
    return q[3] > 0 && fabs(q[0]) <= kMaxCoord && fabs(q[1]) <= kMaxCoord && fabs(q[2]) <= kMaxCoord;
}

__device__ __forceinline__ double view_b(double y, double z) { return __dmul_rn(__dsub_rn(z, y), kS); }

// the fit of one panel: a = X and b = (Z - Y) S map to pixels x = rint(ox + (a - amin) k), y = rint(oy + (bmax - b) k)
struct Fit {
    double amin, bmax, k, ox, oy;
    __device__ __forceinline__ int px(double v) const { return (int)fmin(fmax(rint(v), (double)-COORD_MAX), (double)COORD_MAX); }
    __device__ __forceinline__ void project(double x, double y, double z, int* u, int* v) const {
        *u = px(__dadd_rn(ox, __dmul_rn(__dsub_rn(x, amin), k)));
        *v = px(__dadd_rn(oy, __dmul_rn(__dsub_rn(bmax, view_b(y, z)), k)));
    }
};

__global__ void __launch_bounds__(SETUP_THREADS) panel_setup_kernel(const PanelImg* __restrict__ imgs, PanelSeg* __restrict__ segs) {
    __shared__ double depth[NLIMB];  // -inf: not drawn
    __shared__ double red[8][SETUP_THREADS / 32];
    __shared__ double lo[8];
    const PanelImg& I = imgs[blockIdx.x];
    const int nl = persons(I.rec) * SMAPB_NL;
    const double(*pose)[SMAPB_NJ][4] = I.rec->pred3d;
    PanelSeg* S = segs + (size_t)blockIdx.x * PANEL_ELEMS;
    // minima of a, b, Y, Z and of their negations (the maxima) over the joints of drawn limbs
    double m[8];
#pragma unroll
    for (int i = 0; i < 8; i++) m[i] = INFINITY;
    for (int i = threadIdx.x; i < nl; i += blockDim.x) {
        const double* A = pose[i / SMAPB_NL][kPairs[i % SMAPB_NL][0]];
        const double* B = pose[i / SMAPB_NL][kPairs[i % SMAPB_NL][1]];
        double d = -INFINITY;
        if (placed(A) && placed(B)) {
            d = __dadd_rn(__dadd_rn(A[1], A[2]), __dadd_rn(B[1], B[2]));
#pragma unroll
            for (int t = 0; t < 2; t++) {
                const double* q = t ? B : A;
                const double v[4] = {q[0], view_b(q[1], q[2]), q[1], q[2]};
#pragma unroll
                for (int c = 0; c < 4; c++) m[c] = fmin(m[c], v[c]), m[4 + c] = fmin(m[4 + c], -v[c]);
            }
        }
        depth[i] = d;
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < 8; c++) {
        for (int o = 16; o; o >>= 1) m[c] = fmin(m[c], __shfl_xor_sync(0xffffffffu, m[c], o));
        if (lane == 0) red[c][wid] = m[c];
    }
    __syncthreads();
    if (threadIdx.x < 8) {
        double v = INFINITY;
        for (int w = 0; w < SETUP_THREADS / 32; w++) v = fmin(v, red[threadIdx.x][w]);
        lo[threadIdx.x] = v;
    }
    __syncthreads();
    const bool any = lo[0] != INFINITY;  // the fit set is not empty
    Fit F;
    F.amin = lo[0], F.bmax = -lo[5];
    const double amax = -lo[4], bmin = lo[1];
    const int P = I.P, mg = P / 20;
    const double avail = P - 1 - 2 * mg;
    const double ea = __dsub_rn(amax, F.amin), eb = __dsub_rn(F.bmax, bmin), span = fmax(ea, eb);
    F.k = span > 0 && avail > 0 ? __ddiv_rn(avail, span) : 0.0;
    if (isinf(F.k)) F.k = 0.0;  // a span so small that avail / span overflows
    F.ox = __dadd_rn(mg, __ddiv_rn(__dsub_rn(avail, __dmul_rn(ea, F.k)), 2.0));
    F.oy = __dadd_rn(mg, __ddiv_rn(__dsub_rn(avail, __dmul_rn(eb, F.k)), 2.0));
    for (int i = threadIdx.x; i < nl; i += blockDim.x) {
        PanelSeg s = {0, 0, 0, 0, 0};
        const double d = depth[i];
        if (d != -INFINITY) {
            int rank = 0;  // the drawn limbs painted before this one: farther, or as far and earlier in (row, limb) order
            for (int j = 0; j < nl; j++) {
                const double e = depth[j];
                rank += e > d || (e == d && j < i);
            }
            const int p = i / SMAPB_NL;
            const double* A = pose[p][kPairs[i % SMAPB_NL][0]];
            const double* B = pose[p][kPairs[i % SMAPB_NL][1]];
            F.project(A[0], A[1], A[2], &s.ax, &s.ay);
            F.project(B[0], B[1], B[2], &s.bx, &s.by);
            s.label = (PANEL_BOX + rank + 1) << 3 | p % 6;
        }
        S[PANEL_BOX + i] = s;
    }
    if (threadIdx.x < PANEL_BOX) {
        const int e = threadIdx.x;
        PanelSeg s = {0, 0, 0, 0, 0};
        if (any) {
            // X = a, Y and Z: bits 0, 1, 2 of the corner pick the maximum (a negated minimum) or the minimum
            const int c0 = kBoxEdges[e][0], c1 = kBoxEdges[e][1];
            F.project(c0 & 1 ? amax : F.amin, c0 & 2 ? -lo[6] : lo[2], c0 & 4 ? -lo[7] : lo[3], &s.ax, &s.ay);
            F.project(c1 & 1 ? amax : F.amin, c1 & 2 ? -lo[6] : lo[2], c1 & 4 ? -lo[7] : lo[3], &s.bx, &s.by);
            s.label = (e + 1) << 3 | PANEL_GREY;
        }
        S[e] = s;
    }
}

__global__ void __launch_bounds__(256) panel_paint_kernel(const PanelImg* __restrict__ imgs, const PanelSeg* __restrict__ segs,
                                                          int* __restrict__ labels) {
    const PanelImg& I = imgs[blockIdx.y];
    if ((int)blockIdx.x >= PANEL_BOX + persons(I.rec) * SMAPB_NL) return;
    const PanelSeg s = segs[(size_t)blockIdx.y * PANEL_ELEMS + blockIdx.x];
    if (!s.label) return;
    paint_band(labels + I.base, I.stride, I.P, I.P, s.ax, s.ay, s.bx, s.by, max(1, I.P / 400), s.label);
}

}  // namespace

void panel_launch(const PanelImg* imgs, int n, PanelSeg* segs, int* labels, cudaStream_t st) {
    panel_setup_kernel<<<n, SETUP_THREADS, 0, st>>>(imgs, segs);
    panel_paint_kernel<<<dim3(PANEL_ELEMS, n), 256, 0, st>>>(imgs, segs, labels);
}

}  // namespace smapb
