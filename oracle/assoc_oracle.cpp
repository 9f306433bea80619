/*
 * ORACLE - TEST INFRASTRUCTURE ONLY.  Not part of the product path.
 *
 * CPU restatement (C-style C++, fp32 with pinned FMA placement) of the SMAP
 * depth-aware part association.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library.
 *
 * Follows, function by function:
 *   oracle_nms      <- extensions/gpu/nmsBase.cu:10-50  (nmsRegisterKernel)
 *                      extensions/gpu/nmsBase.cu:165-166 (thrust::exclusive_scan)
 *                      extensions/gpu/nmsBase.cu:52-135 (writeResultKernel)
 *   oracle_paf      <- extensions/gpu/bodyPartConnectorBase.cu:11-63 (process)
 *                      extensions/gpu/bodyPartConnectorBase.cu:104-150 (pafScoreKernel)
 *   oracle_group    <- extensions/association.cpp:123-233 (findConnectedJoints)
 *   oracle_connect  <- extensions/association.cpp:34-120 + 123-233 composed
 *
 * FMA placement follows the SASS of the unmodified reference build
 * (nvcc default -fmad=true): see SURVEY.md section 8(a) rows B3/B4.  Compile
 * with -ffp-contract=off so that gcc adds no contraction of its own; every
 * fused op below is an explicit fmaf().
 *
 * Parity pin: the reference ships no golden vectors for this path.  This file
 * is pinned on the GPU box against oracle/_ref/dapalib (the UNMODIFIED
 * reference extension compiled from /root/reference/extensions by
 * oracle/build_ref.py) in tests/test_assoc_gpu.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

extern "C" {

#define NJ 15
#define NL 14
#define MAXP 127
#define NC 43

/* association.cpp:23-25 */
static const int kJointPairs[2 * NL] = {0, 1, 0, 2, 0, 9, 9, 10, 10, 11, 0, 3, 3, 4,
                                        4, 5, 2, 12, 12, 13, 13, 14, 2, 6, 6, 7, 7, 8};
/* association.cpp:27-31 (float literals narrowed from double, as vector<float>{...}) */
static const float kBoneLength[NL] = {26.42178982f, 48.36980909f, 14.88291009f, 31.28002332f,
                                      23.915707f,   14.97674918f, 31.28002549f, 23.91570732f,
                                      12.4644364f,  48.26604433f, 39.03553194f, 12.4644364f,
                                      48.19076948f, 39.03553252f};

/* ---------------------------------------------------------------- NMS ---- */
/* peaks: [NJ][MAXP+1][3]; slot 0 = (count, -, -), slots 1..count = (x, y, score)
 * in raster order.  Slots beyond count are left untouched (the reference leaves
 * them uninitialised); callers must zero the buffer if they want determinism. */
void oracle_nms(const float* hms, int h, int w, float threshold, float* peaks) {
    const int hw = h * w;
    uint8_t* flag = (uint8_t*)malloc((size_t)hw);
    for (int c = 0; c < NJ; c++) {
        const float* src = hms + (size_t)c * hw;
        float* out = peaks + (size_t)c * (MAXP + 1) * 3;
        /* nmsBase.cu:24-49: strict 3x3 local maximum above threshold, borders 0 */
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                int f = 0;
                if (0 < x && x < w - 1 && 0 < y && y < h - 1) {
                    const float v = src[y * w + x];
                    if (v > threshold) {
                        f = v > src[(y - 1) * w + x - 1] && v > src[(y - 1) * w + x] &&
                            v > src[(y - 1) * w + x + 1] && v > src[y * w + x - 1] &&
                            v > src[y * w + x + 1] && v > src[(y + 1) * w + x - 1] &&
                            v > src[(y + 1) * w + x] && v > src[(y + 1) * w + x + 1];
                    }
                }
                flag[y * w + x] = (uint8_t)f;
            }
        /* nmsBase.cu:165-166 + 61-63,75: exclusive scan, rebased per channel */
        int running = 0;
        for (int i = 0; i < hw; i++) {
            if (flag[i]) {
                const int peakIndex = running;
                running++;
                if (peakIndex < MAXP) { /* nmsBase.cu:92 */
                    const int px = i % w, py = i / w;
                    float xAcc = 0.f, yAcc = 0.f, sAcc = 0.f;
                    for (int dy = -3; dy <= 3; dy++) {
                        const int y = py + dy;
                        if (0 <= y && y < h)
                            for (int dx = -3; dx <= 3; dx++) {
                                const int x = px + dx;
                                if (0 <= x && x < w) {
                                    const float s = src[y * w + x];
                                    if (s > 0) {
                                        /* nmsBase.cu:112-114; x*score+acc is one FFMA in the
                                         * reference SASS */
                                        xAcc = fmaf((float)x, s, xAcc);
                                        yAcc = fmaf((float)y, s, yAcc);
                                        sAcc += s;
                                    }
                                }
                            }
                    }
                    float* o = out + (peakIndex + 1) * 3;
                    o[0] = xAcc / sAcc + 0.5f; /* nmsBase.cu:124 */
                    o[1] = yAcc / sAcc + 0.5f;
                    o[2] = src[py * w + px];
                }
            }
        }
        out[0] = (float)(running < MAXP ? running : MAXP); /* nmsBase.cu:133 */
    }
    free(flag);
}

/* ---------------------------------------------------------------- PAF ---- */
/* bodyPartConnectorBase.cu:11-63 with T=float */
static float paf_process(const float* a, const float* b, const float* mapX, const float* mapY, int w,
                         int h) {
    const float interThreshold = 0.05f, interMinAboveThreshold = 0.95f, defaultNmsThreshold = 0.1f;
    const float dx = b[0] - a[0];
    const float dy = b[1] - a[1];
    const float dmax = fmaxf(fabsf(dx), fabsf(dy));
    int n = (int)(sqrtf(5 * dmax) + 0.5f);
    n = n < 25 ? n : 25;
    n = n > 5 ? n : 5;
    const float norm = sqrtf(fmaf(dx, dx, dy * dy));
    if ((double)norm > 1e-6) {
        const float sX = a[0], sY = a[1];
        const float ux = dx / norm, uy = dy / norm;
        float sum = 0.f;
        int count = 0;
        const float stepX = dx / (float)n, stepY = dy / (float)n;
        for (int lm = 0; lm < n; lm++) {
            int mX = (int)(fmaf((float)lm, stepX, sX) + 0.5f);
            int mY = (int)(fmaf((float)lm, stepY, sY) + 0.5f);
            mX = mX < w - 1 ? mX : w - 1;
            mY = mY < h - 1 ? mY : h - 1;
            const int idx = mY * w + mX;
            const float score = fmaf(ux, mapX[idx], uy * mapY[idx]);
            if (score > interThreshold) {
                sum += score;
                count++;
            }
        }
        if ((float)count / (float)n > interMinAboveThreshold) return sum / (float)count;
        /* bodyPartConnectorBase.cu:56-59; l2Dist is CSE'd with norm in the reference binary */
        const float threshold = sqrtf((float)(w * h)) / 150;
        if (norm < threshold) return (float)(defaultNmsThreshold + 1e-6);
    }
    return -1.f;
}

/* scores: [NL][MAXP][MAXP], fully written (-1 outside nA x nB) as pafScoreKernel does. */
void oracle_paf(const float* hms, int h, int w, const float* peaks, float* scores) {
    const int hw = h * w;
    for (int l = 0; l < NL; l++) {
        const int partA = kJointPairs[2 * l], partB = kJointPairs[2 * l + 1];
        const float* pA = peaks + (size_t)partA * (MAXP + 1) * 3;
        const float* pB = peaks + (size_t)partB * (MAXP + 1) * 3;
        const int nA = (int)pA[0], nB = (int)pB[0];
        const float* mapX = hms + (size_t)(NJ + 2 * l) * hw;     /* association.cpp:40-45 */
        const float* mapY = hms + (size_t)(NJ + 2 * l + 1) * hw;
        float* out = scores + (size_t)l * MAXP * MAXP;
        for (int ia = 0; ia < MAXP; ia++)
            for (int ib = 0; ib < MAXP; ib++)
                out[ia * MAXP + ib] = (ia < nA && ib < nB)
                                          ? paf_process(pA + 3 * (ia + 1), pB + 3 * (ib + 1), mapX, mapY, w, h)
                                          : -1.f;
    }
}

/* ----------------------------------------------------------- grouping ---- */
/* association.cpp:123-233.  bodies: [MAXP][NJ][4] (zeroed here); returns P. */
int oracle_group(const float* peaks, const float* scores, const float* rdepth, int h, int w, int rootIdx,
                 int distFlag, float* bodies) {
    (void)h;
    const float dsScale = 4.f; /* association.cpp:22 */
    const float* rootPeaks = peaks + (size_t)rootIdx * (MAXP + 1) * 3;
    const int P = (int)rootPeaks[0];
    memset(bodies, 0, sizeof(float) * MAXP * NJ * 4);
    if (P == 0) return 0; /* association.cpp:133-136 */

    float depth[MAXP];
    int order[MAXP];
    for (int i = 0; i < P; i++) { /* association.cpp:139-142: int truncation of (y, x) */
        const int yy = (int)rootPeaks[3 * (i + 1) + 1], xx = (int)rootPeaks[3 * (i + 1)];
        depth[i] = rdepth[yy * w + xx];
        order[i] = i;
    }
    /* association.cpp:144 `predRootDepth.sort(0, false)`: at::sort with stable=false on a CPU tensor is
     * std::sort over (key, index) pairs with the comparator below (ATen SortingKernel.cpp, KeyValueCompAsc).
     * It is NOT stable; the order of equal depths is whatever libstdc++'s introsort leaves, which is
     * deterministic and is verified against torch.sort in tests/test_oracle_assoc.py. */
    {
        struct KV {
            float k;
            int v;
        };
        KV kv[MAXP];
        for (int i = 0; i < P; i++) {
            kv[i].k = depth[i];
            kv[i].v = i;
        }
        std::sort(kv, kv + P, [](const KV& a, const KV& b) { return (!std::isnan(a.k) && std::isnan(b.k)) || (a.k < b.k); });
        for (int i = 0; i < P; i++) order[i] = kv[i].v;
    }
    float sortDepth[MAXP];
    for (int i = 0; i < P; i++) sortDepth[i] = depth[order[i]];

    int remap[NJ][MAXP]; /* association.cpp:148-154 */
    for (int j = 0; j < NJ; j++)
        for (int p = 0; p < P; p++) remap[j][p] = (j == rootIdx) ? order[p] : p;

    for (int p = 0; p < P; p++) { /* association.cpp:156-162 */
        const float* pk = rootPeaks + 3 * (order[p] + 1);
        float* b = bodies + ((size_t)p * NJ + rootIdx) * 4;
        b[0] = pk[0];
        b[1] = pk[1];
        b[3] = pk[2];
    }

    for (int j = 0; j < NL; j++) {
        const int i = (j == 0) ? 1 : (j == 1) ? 0 : j; /* association.cpp:167-170 */
        int src, dst, flip = 0;
        if (rootIdx == 2 && i == 1) { /* association.cpp:171-174 */
            src = kJointPairs[2 * i + 1];
            dst = kJointPairs[2 * i];
            flip = 1;
        } else {
            src = kJointPairs[2 * i];
            dst = kJointPairs[2 * i + 1];
        }
        int remapSrc[MAXP];
        memcpy(remapSrc, remap[src], sizeof(int) * P); /* copy taken before the limb is processed */
        const float* dstPeaks = peaks + (size_t)dst * (MAXP + 1) * 3;
        const int dstSize = (int)dstPeaks[0];
        if (dstSize == 0) continue;
        const float* sc = scores + (size_t)i * MAXP * MAXP;
        uint8_t used[MAXP];
        memset(used, 0, sizeof(used));
        for (int k1 = 0; k1 < P; k1++) {
            const float* s = bodies + ((size_t)k1 * NJ + src) * 4;
            if ((double)s[3] < 1e-5) continue; /* association.cpp:190 */
            const float sx = s[0], sy = s[1];
            const float bone_dist = (float)(1.2 * (double)kBoneLength[i] / (double)sortDepth[k1]);
            float maxScore = 0.0f;
            int maxIdx = -1;
            for (int k2 = 0; k2 < dstSize; k2++) {
                if (used[k2]) continue;
                float score = flip ? sc[k2 * MAXP + remapSrc[k1]] : sc[remapSrc[k1] * MAXP + k2];
                if (distFlag && score > 0) {
                    const float ddx = sx - dstPeaks[3 * (k2 + 1)], ddy = sy - dstPeaks[3 * (k2 + 1) + 1];
                    const float limb_dist =
                        (float)sqrt((double)ddx * (double)ddx + (double)ddy * (double)ddy);
                    const float t = bone_dist / limb_dist / dsScale - 1; /* association.cpp:211 */
                    const float z = 0.0f;
                    score += (z < t) ? z : t; /* std::min(t, 0.0f) */
                }
                if (score > maxScore) {
                    maxScore = score;
                    maxIdx = k2;
                }
            }
            if (maxScore > 0) { /* association.cpp:220-228 */
                float* d = bodies + ((size_t)k1 * NJ + dst) * 4;
                d[0] = dstPeaks[3 * (maxIdx + 1)];
                d[1] = dstPeaks[3 * (maxIdx + 1) + 1];
                d[3] = dstPeaks[3 * (maxIdx + 1) + 2];
                remap[dst][k1] = maxIdx;
                used[maxIdx] = 1;
            }
        }
    }
    return P;
}

/* dapalib.connect equivalent for one image.  hms [43][h][w] already /255,/127.
 * peaks [NJ][128][3] and scores [NL][127][127] are scratch/outputs supplied by the caller. */
int oracle_connect(const float* hms, const float* rdepth, int h, int w, int rootIdx, int distFlag,
                   float* peaks, float* scores, float* bodies) {
    memset(peaks, 0, sizeof(float) * NJ * (MAXP + 1) * 3);
    oracle_nms(hms, h, w, 0.2f, peaks);
    oracle_paf(hms, h, w, peaks, scores);
    return oracle_group(peaks, scores, rdepth, h, w, rootIdx, distFlag, bodies);
}

/* test hook: the sort of association.cpp:144 alone (order[i] = index of the i-th smallest depth) */
void oracle_depth_order(const float* depth, int n, int* order) {
    struct KV {
        float k;
        int v;
    };
    KV* kv = new KV[n];
    for (int i = 0; i < n; i++) {
        kv[i].k = depth[i];
        kv[i].v = i;
    }
    std::sort(kv, kv + n, [](const KV& a, const KV& b) { return (!std::isnan(a.k) && std::isnan(b.k)) || (a.k < b.k); });
    for (int i = 0; i < n; i++) order[i] = kv[i].v;
    delete[] kv;
}

} /* extern "C" */
