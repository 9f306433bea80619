// Exact integer coverage tests and the band walk that paints one skeleton element into a label plane, shared by the
// frame overlay (jpeg_enc.cu) and the 3D panel (view3d.cu) of the JPEG encoder.
#pragma once
#include <math.h>

#include "../../include/smap_b200.h"

namespace smapb {

// the 14 limbs: joint pairs of lib/preprocess/data_format.md
static __constant__ int kPairs[SMAPB_NL][2] = {{0, 1}, {0, 2}, {0, 9}, {9, 10}, {10, 11}, {0, 3}, {3, 4},
                                               {4, 5}, {2, 12}, {12, 13}, {13, 14}, {2, 6}, {6, 7}, {7, 8}};

constexpr int COORD_MAX = 32768;  // element coordinates are clamped to +-COORD_MAX (so the limb test fits int64)

__device__ __forceinline__ bool in_disc(long long dx, long long dy, long long rr) { return dx * dx + dy * dy <= rr * rr; }

// clamped-projection test of pixel (x, y) against the limb a-b of half-width r, exact in int64
__device__ __forceinline__ bool in_limb(long long x, long long y, long long ax, long long ay, long long bx, long long by, long long r) {
    const long long vx = bx - ax, vy = by - ay, px = x - ax, py = y - ay;
    const long long dot = px * vx + py * vy, len2 = vx * vx + vy * vy;
    if (dot <= 0) return in_disc(px, py, r);
    if (dot >= len2) return in_disc(x - bx, y - by, r);
    const long long cross = px * vy - py * vx;
    if (cross > (1ll << 31) || cross < -(1ll << 31)) return false;  // cross^2 > 2^62 > r^2 |b-a|^2
    return cross * cross <= r * r * len2;
}

// One CTA atomicMax-es `rank` into L[y * stride + x] for every pixel of [0, w) x [0, h) that the limb a-b of half-width
// rad covers; a joint is a limb a = b, tested as a disc.
// Candidates: along the segment's major axis, its range widened by rad; across it, a band of +-(2 rad + 2) around the
// segment's (clamped, rounded) centre line.  A covered pixel is within rad of some segment point, so within
// sqrt(2) rad + 1/2 of that line across the major axis: the band holds every pixel the exact test accepts, and a long
// diagonal limb costs its length times the band instead of its bounding box.
__device__ __forceinline__ void paint_band(int* L, long long stride, long long w, long long h, long long ax, long long ay,
                                           long long bx, long long by, long long rad, int rank) {
    const bool disc = ax == bx && ay == by;
    const bool xmajor = llabs(bx - ax) >= llabs(by - ay);
    const long long am = xmajor ? ax : ay, bm = xmajor ? bx : by, an = xmajor ? ay : ax, bn = xmajor ? by : bx;
    const long long lim_m = xmajor ? w : h, lim_n = xmajor ? h : w;
    const long long m0 = max(0ll, min(am, bm) - rad), m1 = min(lim_m - 1, max(am, bm) + rad);
    if (m0 > m1) return;
    const long long band = 2 * rad + 2, span = 2 * band + 1, count = (m1 - m0 + 1) * span;
    for (long long k = threadIdx.x; k < count; k += blockDim.x) {
        const long long m = m0 + k / span;
        const long long mc = min(max(m, min(am, bm)), max(am, bm));
        const long long c = bm == am ? an : (long long)rint(an + (double)(mc - am) * (double)(bn - an) / (double)(bm - am));
        const long long nn = c + k % span - band;
        if (nn < 0 || nn >= lim_n) continue;
        const long long x = xmajor ? m : nn, y = xmajor ? nn : m;
        const bool hit = disc ? in_disc(x - ax, y - ay, rad) : in_limb(x, y, ax, ay, bx, by, rad);
        if (hit) atomicMax(&L[y * stride + x], rank);
    }
}

}  // namespace smapb
