// Depth-aware part association on sm_90a: batched, device-resident, bit-exact with the reference.
//
//   nms_kernel    <- extensions/gpu/nmsBase.cu:10-135 (register + thrust scan + write, fused)
//   paf_kernel    <- extensions/gpu/bodyPartConnectorBase.cu:11-63,104-150
//   group_kernel  <- extensions/association.cpp:123-233 (findConnectedJoints; CPU in the reference)
//   lift_kernel   <- exps/stage3_root2/test_util.py:60-99 + lib/utils/post_3d.py:4-27 (numpy in the reference)
//
// Data movement: every heat-map / PAF plane is staged ONCE into shared memory with 1-D bulk async copies
// (cp.async.bulk -> UBLKCP, completion on an mbarrier); all neighbourhood / line-integral gathers then hit
// shared memory.  Floating-point expressions whose rounding feeds a comparison are pinned with explicit
// __f*_rn intrinsics in the contraction pattern of the reference's binary (SURVEY.md 8(a) B3/B4).
#include "assoc.h"
#include "common.cuh"

namespace smapb {

__constant__ int c_joint_pairs[2 * NL] = {0, 1, 0, 2, 0, 9, 9, 10, 10, 11, 0, 3, 3, 4,
                                          4, 5, 2, 12, 12, 13, 13, 14, 2, 6, 6, 7, 7, 8};
// extensions/association.cpp:27-31 (vector<float> initialised from double literals)
__constant__ float c_bone_length[NL] = {26.42178982f, 48.36980909f, 14.88291009f, 31.28002332f, 23.915707f,
                                        14.97674918f, 31.28002549f, 23.91570732f, 12.4644364f, 48.26604433f,
                                        39.03553194f, 12.4644364f, 48.19076948f, 39.03553252f};

// ---------------------------------------------------------------------------------------------
// NMS in two streaming passes (replaces nmsRegisterKernel + thrust::exclusive_scan + writeResultKernel,
// extensions/gpu/nmsBase.cu:10-135), for any map size:
//   nms_flag_kernel    : every warp tests 32 consecutive pixels of a plane per step (3x3 strict maximum above the
//                        threshold, borders excluded) and stores the ballot word - one coalesced 128-byte read per step,
//                        the 8 neighbours are only fetched for the few pixels above the threshold.  Pure HBM stream:
//                        the planes are read exactly once, the bit masks (h*w/8 bytes per plane) are the only output.
//   nms_compact_kernel : one CTA per (image, key-point channel) turns the bit mask into the raster-ordered peak list
//                        (popcount prefix over contiguous runs of words = the reference's global exclusive scan restricted
//                        to the plane, nmsBase.cu:165-166 + :57-60) and refines each peak with the 7x7 score-weighted
//                        centroid (nmsBase.cu:84-133) - the 49 taps come from L2, which the flag pass has just filled.
// Peak order is raster order: candidate indices are part of the parity contract.
// ---------------------------------------------------------------------------------------------
constexpr int NMSF_THREADS = 256;
constexpr int NMSC_THREADS = 256;
constexpr int NMSC_WARPS = NMSC_THREADS / 32;

// strict 3x3 maximum above the threshold, borders excluded (nmsBase.cu:24-49); v = plane[i] is already known to be > thr
__device__ __forceinline__ bool nms_is_peak(const float* __restrict__ plane, int i, float v, int h, int w) {
    const int y = i / w, x = i - y * w;
    if (!(x > 0 && x < w - 1 && y > 0 && y < h - 1)) return false;
    const float* q0 = plane + i - w;
    const float* q2 = plane + i + w;
    // all eight neighbours are requested before the first comparison (no short-circuit: one memory latency, not eight)
    const float n0 = __ldg(q0 - 1), n1 = __ldg(q0), n2 = __ldg(q0 + 1), n3 = __ldg(plane + i - 1), n4 = __ldg(plane + i + 1),
                n5 = __ldg(q2 - 1), n6 = __ldg(q2), n7 = __ldg(q2 + 1);
    return (v > n0) & (v > n1) & (v > n2) & (v > n3) & (v > n4) & (v > n5) & (v > n6) & (v > n7);
}

// VEC: h*w % 128 == 0 - a warp step covers 2 x 128 consecutive pixels with two 16-byte loads per lane in flight (1 KB
// per warp per step: enough requests outstanding to keep HBM busy; the scalar variant handles any other map size).
template <bool VEC>
__global__ void __launch_bounds__(NMSF_THREADS)
nms_flag_kernel(const float* __restrict__ hms, int nchan, int B, int h, int w, float thr, uint32_t* __restrict__ masks) {
    const int hw = h * w;
    const int nwords = (hw + 31) / 32;
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    if (VEC) {
        // persistent: one wave of CTAs, every warp strides over 4-group (512-pixel, 2 KB) steps with all four 16-byte
        // loads of a lane in flight before any of them is consumed.  Pixels above the threshold (candidates) are NOT
        // tested where they are found - a lane that meets one would stall the other 31 on eight neighbour loads, and the
        // next lane would do the same a few instructions later: instead the warp collects the step's candidates in a small
        // shared list and tests them side by side, one candidate per lane (one memory latency per 32 candidates).
        constexpr int U = 4;
        __shared__ uint32_t s_words[NMSF_THREADS / 32][4 * U];
        __shared__ int s_cand[NMSF_THREADS / 32][64];   // (u << 16) | pixel offset inside the 128-pixel group ... | k
        __shared__ float s_val[NMSF_THREADS / 32][64];
        const int wl = threadIdx.x >> 5;
        const int groups = hw / 128;                       // 128-pixel groups per plane (4 ballot words each)
        const int total = B * NJ * groups;                 // < 2^31 for any batch that fits the workspace
        for (int g0 = (int)warp0 * U; g0 < total; g0 += (int)nwarps * U) {
            float4 v[U];
            const float* pl[U];
            int gi[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int g = g0 + u;
                const bool ok = g < total;
                const int plane_id = ok ? g / groups : 0;
                gi[u] = ok ? g - plane_id * groups : 0;
                const int img = plane_id / NJ, c = plane_id - img * NJ;
                pl[u] = hms + ((size_t)img * nchan + c) * hw;
                v[u] = ok ? __ldg(reinterpret_cast<const float4*>(pl[u] + gi[u] * 128 + lane * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if (lane < 4 * U) s_words[wl][lane] = 0u;
            // candidate bits of this lane: bit (u * 4 + k)
            uint32_t cbits = 0;
#pragma unroll
            for (int u = 0; u < U; u++) {
                const float vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if (vv[k] > thr) cbits |= 1u << (u * 4 + k);
            }
            __syncwarp();
            uint32_t pending = cbits;
            while (__any_sync(0xffffffffu, pending != 0)) {
                // warp-wide exclusive scan of the candidate counts -> list positions; a round takes at most 64 entries
                const int mine = __popc(pending);
                int incl = mine;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int n = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += n;
                }
                int pos = incl - mine;
                const int n_all = __shfl_sync(0xffffffffu, incl, 31);
                uint32_t rest = pending;
                while (rest && pos < 64) {
                    const int bit = __ffs(rest) - 1;
                    rest &= rest - 1;
                    const int u = bit >> 2, k = bit & 3;
                    s_cand[wl][pos] = (u << 16) | (lane * 4 + k);
                    float val = 0.f;
#pragma unroll
                    for (int uu = 0; uu < U; uu++) {
                        const float vv[4] = {v[uu].x, v[uu].y, v[uu].z, v[uu].w};
#pragma unroll
                        for (int kk = 0; kk < 4; kk++)
                            if (uu == u && kk == k) val = vv[kk];
                    }
                    s_val[wl][pos] = val;
                    pos++;
                }
                pending = rest;  // whatever did not fit waits for the next round
                __syncwarp();
                const int n_round = n_all < 64 ? n_all : 64;
                for (int e = lane; e < n_round; e += 32) {
                    const int ent = s_cand[wl][e];
                    const int u = ent >> 16, off = ent & 0xffff;
                    // pl[] / gi[] are the same in every lane: pick entry u without dynamic register indexing
                    const float* plane = u == 0 ? pl[0] : u == 1 ? pl[1] : u == 2 ? pl[2] : pl[3];
                    const int gidx = u == 0 ? gi[0] : u == 1 ? gi[1] : u == 2 ? gi[2] : gi[3];
                    if (nms_is_peak(plane, gidx * 128 + off, s_val[wl][e], h, w))
                        atomicOr(&s_words[wl][u * 4 + (off >> 5)], 1u << (off & 31));
                }
                __syncwarp();
            }
            if (lane < 4 * U && g0 + (lane >> 2) < total) masks[(size_t)g0 * 4 + lane] = s_words[wl][lane];  // nwords == 4 * groups
            __syncwarp();
        }
    } else {
        const long long total = (long long)B * NJ * nwords;  // ballot words of all planes
        for (long long wd = warp0; wd < total; wd += nwarps) {
            const int plane_id = (int)(wd / nwords), wi = (int)(wd - (long long)plane_id * nwords);
            const int img = plane_id / NJ, c = plane_id - img * NJ;
            const float* plane = hms + ((size_t)img * nchan + c) * hw;
            const int i = wi * 32 + lane;
            bool f = false;
            if (i < hw) {
                const float v = __ldg(plane + i);
                f = v > thr && nms_is_peak(plane, i, v, h, w);
            }
            const uint32_t m = __ballot_sync(0xffffffffu, f);
            if (lane == 0) masks[wd] = m;
        }
    }
}

__global__ void __launch_bounds__(NMSC_THREADS)
nms_compact_kernel(const float* __restrict__ hms, int nchan, int h, int w, const uint32_t* __restrict__ masks,
                   float* __restrict__ peaks) {
    __shared__ int warp_tot[NMSC_WARPS];
    const int hw = h * w;
    const int nwords = (hw + 31) / 32;
    const int c = blockIdx.x, img = blockIdx.y;
    const float* plane = hms + ((size_t)img * nchan + c) * hw;
    const uint32_t* mk = masks + ((size_t)img * NJ + c) * nwords;
    float* out = peaks + ((size_t)img * NJ + c) * (MAXP + 1) * 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // contiguous run of words per warp, lanes stride through the run; counts first
    const int wpw = (nwords + NMSC_WARPS - 1) / NMSC_WARPS;
    const int w0 = min(nwords, warp * wpw), w1 = min(nwords, w0 + wpw);
    int cnt = 0;
    for (int wi = w0 + lane; wi < w1; wi += 32) cnt += __popc(__ldg(mk + wi));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) warp_tot[warp] = cnt;
    __syncthreads();
    int t = (lane < NMSC_WARPS) ? warp_tot[lane] : 0;
    int before = (lane < warp) ? t : 0;
    int total = t;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        before += __shfl_xor_sync(0xffffffffu, before, o);
        total += __shfl_xor_sync(0xffffffffu, total, o);
    }
    // the warp walks its run 32 words at a time: an in-warp exclusive scan of the word popcounts gives every word its
    // first peak index, then each lane expands its own word (peaks are sparse: a word rarely holds more than one)
    int running = before;
    for (int base = w0; base < w1 && running < MAXP; base += 32) {
        const int wi = base + lane;
        const uint32_t m = (wi < w1) ? __ldg(mk + wi) : 0u;
        const int pc = __popc(m);
        int incl = pc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += n;
        }
        int peakIndex = running + incl - pc;
        uint32_t mm = m;
        while (mm) {
            const int bit = __ffs(mm) - 1;
            mm &= mm - 1;
            if (peakIndex < MAXP) {  // nmsBase.cu:92
                const int i = wi * 32 + bit;
                const int py = i / w, px = i - py * w;
                float xAcc = 0.f, yAcc = 0.f, sAcc = 0.f;
                // all 49 taps are requested before the first one is used (one memory latency per peak instead of seven:
                // at B = 64 the planes have left L2 by the time this kernel runs), then accumulated in the reference's
                // order (dy outer, dx inner; nmsBase.cu:101-117)
                float tap[7][7];
#pragma unroll
                for (int dy = 0; dy < 7; dy++) {
                    const int y = py + dy - 3;
#pragma unroll
                    for (int dx = 0; dx < 7; dx++) {
                        const int x = px + dx - 3;
                        tap[dy][dx] = (y >= 0 && y < h && x >= 0 && x < w) ? __ldg(plane + y * w + x) : 0.f;  // outside: skipped like s <= 0
                    }
                }
#pragma unroll
                for (int dy = 0; dy < 7; dy++) {
#pragma unroll
                    for (int dx = 0; dx < 7; dx++) {
                        const float sc = tap[dy][dx];
                        if (sc > 0) {
                            xAcc = __fmaf_rn((float)(px + dx - 3), sc, xAcc);  // FFMA in the reference SASS
                            yAcc = __fmaf_rn((float)(py + dy - 3), sc, yAcc);
                            sAcc = __fadd_rn(sAcc, sc);
                        }
                    }
                }
                float* o = out + (peakIndex + 1) * 3;
                o[0] = __fadd_rn(__fdiv_rn(xAcc, sAcc), 0.5f);
                o[1] = __fadd_rn(__fdiv_rn(yAcc, sAcc), 0.5f);
                o[2] = __ldg(plane + i);
            }
            peakIndex++;
        }
        running += __shfl_sync(0xffffffffu, incl, 31);
    }
    const int count = total < MAXP ? total : MAXP;
    if (threadIdx.x == 0) {
        out[0] = (float)count;
        out[1] = 0.f;
        out[2] = 0.f;
    }
    // deterministic tail: slots the reference leaves uninitialised are zeroed
    for (int k = (count + 1) * 3 + threadIdx.x; k < (MAXP + 1) * 3; k += NMSC_THREADS) out[k] = 0.f;
}

// ---------------------------------------------------------------------------------------------
// PAF line-integral scoring: one CTA per (image, limb); both PAF planes (adjacent channels 15+2l, 16+2l)
// are staged once into shared memory, then one thread per (peakA, peakB) candidate.
// ---------------------------------------------------------------------------------------------
constexpr int PAF_THREADS = 1024;

// `sample(idx, px, py)` returns the two PAF components at pixel idx (shared memory, peer shared memory or global memory)
template <typename Sampler>
__device__ __forceinline__ float paf_process(float ax, float ay, float bx, float by, const Sampler& sample, int w, int h,
                                             float near_thr) {
    const float dx = __fsub_rn(bx, ax);
    const float dy = __fsub_rn(by, ay);
    const float dmax = fmaxf(fabsf(dx), fabsf(dy));
    int n = (int)__fadd_rn(__fsqrt_rn(__fmul_rn(5.f, dmax)), 0.5f);
    n = max(5, min(25, n));
    const float norm = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    if ((double)norm > 1e-6) {
        const float ux = __fdiv_rn(dx, norm), uy = __fdiv_rn(dy, norm);
        const float fn = (float)n;
        const float stepX = __fdiv_rn(dx, fn), stepY = __fdiv_rn(dy, fn);
        float sum = 0.f;
        int count = 0;
        for (int lm = 0; lm < n; lm++) {
            const float flm = (float)lm;
            int mX = (int)__fadd_rn(__fmaf_rn(flm, stepX, ax), 0.5f);
            int mY = (int)__fadd_rn(__fmaf_rn(flm, stepY, ay), 0.5f);
            mX = min(w - 1, mX);
            mY = min(h - 1, mY);
            // the reference applies no lower clamp (coordinates are >= 0.5 by construction); clamp to keep
            // the access in range for adversarial inputs without changing valid results
            mX = max(0, mX);
            mY = max(0, mY);
            float px, py;
            sample(mY * w + mX, px, py);
            const float score = __fmaf_rn(ux, px, __fmul_rn(uy, py));
            if (score > 0.05f) {
                sum = __fadd_rn(sum, score);
                count++;
            }
        }
        if (__fdiv_rn((float)count, fn) > 0.95f) return __fdiv_rn(sum, (float)count);
        if (norm < near_thr) return (float)(0.1f + 1e-6);
    }
    return -1.f;
}

struct PafSamplerPlanes {  // both planes behind ordinary pointers (shared or global memory)
    const float* x;
    const float* y;
    __device__ __forceinline__ void operator()(int idx, float& px, float& py) const {
        px = x[idx];
        py = y[idx];
    }
};
// STAGED: both planes fit in shared memory (the parity configuration 128x208: 213 KB) and are staged once; otherwise
// (larger maps, e.g. 256x256 at a 1024x1024 input) the line integrals gather straight from global memory / L2.
// Two restructurings were built and dropped (timed at B = 64 crowded scenes on the GPU this kernel was first written for):
//  * a cluster of two CTAs per item, one plane each, the other component read through distributed shared memory, so that
//    two CTAs fit on an SM and one's copy overlaps the other's scoring: 78.5 us - 25 dependent DSMEM loads per pair;
//  * a persistent CTA with the x and y planes in separate buffers and the scoring split in an x pass and a y pass, so that
//    a plane is refilled while the other is in use: 57 - 60 us - the scoring of an item (IEEE sqrt / divisions of the
//    reference, a <= 25-sample chain per pair, CTA barriers) takes longer than its planes
//    need to arrive, so the copy engine was never the bottleneck of this kernel at 15 persons per frame.
template <bool STAGED>
__global__ void __launch_bounds__(PAF_THREADS, 1)
paf_kernel(const float* __restrict__ hms, int nchan, int h, int w, const float* __restrict__ peaks,
           float* __restrict__ scores, int dense_fill) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int hw = h * w;
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
    float* pk = reinterpret_cast<float*>(smem_raw + 16);  // [2][MAXP+1][2]  (x, y) of joint A then joint B
    float* planes = pk + 4 * (MAXP + 1);                  // [2][hw] when STAGED (16-byte aligned: 16 + 2048 bytes in)

    const int l = blockIdx.x, img = blockIdx.y;
    const int partA = c_joint_pairs[2 * l], partB = c_joint_pairs[2 * l + 1];
    const float* pA = peaks + ((size_t)img * NJ + partA) * (MAXP + 1) * 3;
    const float* pB = peaks + ((size_t)img * NJ + partB) * (MAXP + 1) * 3;
    float* out = scores + ((size_t)img * NL + l) * MAXP * MAXP;

    const float* src = hms + ((size_t)img * nchan + NJ + 2 * l) * hw;
    // STAGED: the bulk copies of both planes are issued FIRST, before the candidate counts are even known; the counts and the
    // two peak lists (dependent global loads, ~1 us each) then arrive while the copy engine streams the 213 KB.  An item with
    // an empty peak list has staged its planes for nothing - on a frame that contains people every limb has candidates -
    // but the critical path of an item shrinks from  counts -> planes -> peak lists -> scores  to  planes -> scores
    // (B = 64 crowded scenes).
    if (STAGED) {
        if (threadIdx.x == 0) {
            mbar_init(bar, 1);
            fence_mbar_init();
        }
        __syncthreads();
        // warp 0 issues the copies (one 16 KB chunk per lane per round: up to 32 in flight per CTA) and is the ONLY warp
        // that polls the mbarrier; everyone else parks on the CTA barrier.  (Round 1 had one thread issue 32 KB chunks while
        // all 1024 threads spun on mbarrier.try_wait: the polling traffic slowed the very shared-memory writes it was
        // waiting for - 15 GB/s per SM.)
        if (threadIdx.x < 32) {
            const uint32_t bytes = (uint32_t)hw * 8u;
            if (threadIdx.x == 0) mbar_arrive_expect_tx(bar, bytes);
            __syncwarp();
            const uint32_t CH = 16384;
            for (uint32_t off = threadIdx.x * CH; off < bytes; off += 32 * CH)
                bulk_g2s((char*)planes + off, (const char*)src + off, bytes - off < CH ? bytes - off : CH, bar);
        }
    }
    const int nA = (int)pA[0], nB = (int)pB[0];
    for (int i = threadIdx.x; i < nA; i += PAF_THREADS) {
        pk[2 * i] = pA[3 * (i + 1)];
        pk[2 * i + 1] = pA[3 * (i + 1) + 1];
    }
    for (int i = threadIdx.x; i < nB; i += PAF_THREADS) {
        pk[2 * (MAXP + 1) + 2 * i] = pB[3 * (i + 1)];
        pk[2 * (MAXP + 1) + 2 * i + 1] = pB[3 * (i + 1) + 1];
    }
    if (STAGED && threadIdx.x < 32) mbar_wait(bar, 0);  // (also for an empty item: the copies must land before the CTA retires)
    __syncthreads();
    if (nA > 0 && nB > 0) {
        const float* mapX = STAGED ? planes : src;
        const float near_thr = __fdiv_rn(__fsqrt_rn((float)(w * h)), 150.f);
        const int npairs = nA * nB;
        for (int p = threadIdx.x; p < npairs; p += PAF_THREADS) {
            const int a = p / nB, b = p - a * nB;
            out[a * MAXP + b] = paf_process(pk[2 * a], pk[2 * a + 1], pk[2 * (MAXP + 1) + 2 * b],
                                            pk[2 * (MAXP + 1) + 2 * b + 1], PafSamplerPlanes{mapX, mapX + hw}, w, h, near_thr);
        }
    }
    if (dense_fill) {  // pafScoreKernel writes -1 outside nA x nB; only the extract() API needs it
        for (int p = threadIdx.x; p < MAXP * MAXP; p += PAF_THREADS) {
            const int a = p / MAXP, b = p - a * MAXP;
            if (a >= nA || b >= nB) out[p] = -1.f;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// `predRootDepth.sort(0, false)` (association.cpp:144): at::sort(stable=false) on a CPU tensor is libstdc++
// std::sort over (key, index) pairs with comp(a,b) = (!isnan(a) && isnan(b)) || a < b.  It is not stable, so
// equal depths come out in introsort order.  When all depths are distinct the order is unique and a parallel
// rank sort is used; otherwise one thread replays libstdc++'s algorithm (bits/stl_algo.h: introsort loop with
// median-of-3 to first + unguarded partition, threshold 16, heap-sort fallback at depth 2*floor(log2 n), final
// insertion sort) step by step so that the tie order is bit-identical to the reference.
// ---------------------------------------------------------------------------------------------
struct KV {
    float k;
    int v;
};
__device__ __forceinline__ bool kv_comp(const KV& a, const KV& b) { return (!isnan(a.k) && isnan(b.k)) || (a.k < b.k); }
__device__ __forceinline__ void kv_swap(KV& a, KV& b) {
    const KV t = a;
    a = b;
    b = t;
}
__device__ void kv_adjust_heap(KV* first, int hole, int len, KV value) {  // std::__adjust_heap + __push_heap
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (kv_comp(first[child], first[child - 1])) child--;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    int parent = (hole - 1) / 2;
    while (hole > top && kv_comp(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}
__device__ void kv_heap_sort(KV* first, int len) {  // std::__partial_sort(first, last, last)
    if (len >= 2) {                                  // __make_heap
        int parent = (len - 2) / 2;
        while (true) {
            const KV value = first[parent];
            kv_adjust_heap(first, parent, len, value);
            if (parent == 0) break;
            parent--;
        }
    }
    // __heap_select(first, last, last) has an empty tail; then __sort_heap
    for (int last = len; last > 1;) {
        --last;
        const KV value = first[last];  // __pop_heap(first, last, last)
        first[last] = first[0];
        kv_adjust_heap(first, 0, last, value);
    }
}
__device__ __forceinline__ void kv_unguarded_linear_insert(KV* a, int last) {
    const KV val = a[last];
    int next = last - 1;
    while (kv_comp(val, a[next])) {
        a[last] = a[next];
        last = next;
        --next;
    }
    a[last] = val;
}
__device__ void kv_insertion_sort(KV* a, int first, int last) {
    if (first == last) return;
    for (int i = first + 1; i != last; ++i) {
        if (kv_comp(a[i], a[first])) {
            const KV val = a[i];
            for (int j = i; j > first; --j) a[j] = a[j - 1];
            a[first] = val;
        } else {
            kv_unguarded_linear_insert(a, i);
        }
    }
}
__device__ void kv_std_sort(KV* a, int n) {
    if (n <= 0) return;
    int lg = 0;
    while ((1 << (lg + 1)) <= n) lg++;
    // explicit stack for the recursive half of __introsort_loop
    int st_first[32], st_last[32], st_depth[32];
    int sp = 0;
    st_first[0] = 0, st_last[0] = n, st_depth[0] = 2 * lg;
    sp = 1;
    while (sp > 0) {
        --sp;
        int first = st_first[sp], last = st_last[sp], depth = st_depth[sp];
        while (last - first > 16) {
            if (depth == 0) {
                kv_heap_sort(a + first, last - first);
                break;
            }
            --depth;
            // __unguarded_partition_pivot
            const int mid = first + (last - first) / 2;
            {
                const int ia = first + 1, ib = mid, ic = last - 1;
                if (kv_comp(a[ia], a[ib])) {
                    if (kv_comp(a[ib], a[ic])) kv_swap(a[first], a[ib]);
                    else if (kv_comp(a[ia], a[ic])) kv_swap(a[first], a[ic]);
                    else kv_swap(a[first], a[ia]);
                } else if (kv_comp(a[ia], a[ic])) kv_swap(a[first], a[ia]);
                else if (kv_comp(a[ib], a[ic])) kv_swap(a[first], a[ic]);
                else kv_swap(a[first], a[ib]);
            }
            int lo = first + 1, hi = last;
            while (true) {
                while (kv_comp(a[lo], a[first])) ++lo;
                --hi;
                while (kv_comp(a[first], a[hi])) --hi;
                if (!(lo < hi)) break;
                kv_swap(a[lo], a[hi]);
                ++lo;
            }
            const int cut = lo;
            // recurse on [cut, last), iterate on [first, cut): libstdc++ runs the right part first, but the two
            // ranges are disjoint, so the order of processing does not change the result
            st_first[sp] = cut, st_last[sp] = last, st_depth[sp] = depth;
            ++sp;
            last = cut;
        }
    }
    // __final_insertion_sort
    if (n > 16) {
        kv_insertion_sort(a, 0, 16);
        for (int i = 16; i != n; ++i) kv_unguarded_linear_insert(a, i);
    } else {
        kv_insertion_sort(a, 0, n);
    }
}

// ---------------------------------------------------------------------------------------------
// Grouping: one CTA (5 warps) per image.  The 14 limbs form 5 independent chains hanging off the
// pelvis/neck (dst joints are disjoint, `used` is per limb), so the sequential reference order
//   1,0,2,3,...,13  (association.cpp:164-170)
// is reproduced exactly by running the chains concurrently in 4 barrier-separated phases:
//   phase0: 1 | 8 | 11      phase1: 0 | 2 | 5 | 9 | 12      phase2: 3 | 6 | 10 | 13      phase3: 4 | 7
// Within a limb, persons are visited serially in ascending root depth (the ordinal prior); the scan over
// destination candidates is a warp arg-max with "first index wins" (strict > in ascending k2).
// ---------------------------------------------------------------------------------------------
constexpr int GROUP_WARPS = 5;
__constant__ int c_phase_limb[4][GROUP_WARPS] = {
    {1, -1, -1, 8, 11}, {0, 2, 5, 9, 12}, {-1, 3, 6, 10, 13}, {-1, 4, 7, -1, -1}};
// root_idx != 2 (neck root): the leg chains depend on limb 1, so fall back to the reference's serial order.
__constant__ int c_serial_limb[NL] = {1, 0, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13};

__global__ void __launch_bounds__(GROUP_WARPS * 32, 1)
group_kernel(const float* __restrict__ peaks, const float* __restrict__ scores, const float* __restrict__ rdepth,
             int h, int w, int root_idx, int dist_flag, float* __restrict__ bodies, int* __restrict__ counts) {
    __shared__ float s_depth[MAXP + 1];
    __shared__ float s_sorted[MAXP + 1];
    __shared__ int s_order[MAXP + 1];
    __shared__ int s_rank[MAXP + 1];
    __shared__ unsigned long long s_kv[MAXP + 1];
    __shared__ unsigned char s_remap[NJ][MAXP + 1];
    __shared__ float s_body[MAXP][NJ][3];  // x, y, score
    __shared__ unsigned char s_used[GROUP_WARPS][MAXP + 1];

    const int img = blockIdx.x;
    const float* pk = peaks + (size_t)img * NJ * (MAXP + 1) * 3;
    const float* sc_img = scores + (size_t)img * NL * MAXP * MAXP;
    const float* rd = rdepth + (size_t)img * h * w;
    float* outb = bodies + (size_t)img * MAXP * NJ * 4;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nthr = GROUP_WARPS * 32;

    const float* rootPeaks = pk + (size_t)root_idx * (MAXP + 1) * 3;
    const int P = (int)rootPeaks[0];
    if (tid == 0) counts[img] = P;

    for (int i = tid; i < MAXP * NJ * 3; i += nthr) (&s_body[0][0][0])[i] = 0.f;
    for (int i = tid; i < P; i += nthr) {  // association.cpp:139-142
        const int yy = (int)rootPeaks[3 * (i + 1) + 1], xx = (int)rootPeaks[3 * (i + 1)];
        s_depth[i] = rd[min(h - 1, max(0, yy)) * w + min(w - 1, max(0, xx))];
    }
    __syncthreads();
    // ascending depth order (association.cpp:144): unique keys -> parallel rank sort, ties/NaNs -> std::sort replay
    {
        int tie = 0;
        for (int i = tid; i < P; i += nthr) {
            const KV a = {s_depth[i], i};
            int r = 0;
            for (int j = 0; j < P; j++) {
                const KV b = {s_depth[j], j};
                const bool lt = kv_comp(b, a);
                r += lt;
                tie |= (j != i) && !lt && !kv_comp(a, b);
            }
            s_rank[i] = r;
        }
        const int any_tie = __syncthreads_or(tie);
        if (!any_tie) {
            for (int i = tid; i < P; i += nthr) {
                s_order[s_rank[i]] = i;
                s_sorted[s_rank[i]] = s_depth[i];
            }
        } else if (tid == 0) {
            KV* kv = reinterpret_cast<KV*>(s_kv);
            for (int i = 0; i < P; i++) {
                kv[i].k = s_depth[i];
                kv[i].v = i;
            }
            kv_std_sort(kv, P);
            for (int i = 0; i < P; i++) {
                s_order[i] = kv[i].v;
                s_sorted[i] = kv[i].k;
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < NJ * P; i += nthr) {  // association.cpp:148-154
        const int j = i / P, p = i - j * P;
        s_remap[j][p] = (unsigned char)((j == root_idx) ? s_order[p] : p);
    }
    for (int p = tid; p < P; p += nthr) {  // association.cpp:156-162
        const float* r = rootPeaks + 3 * (s_order[p] + 1);
        s_body[p][root_idx][0] = r[0];
        s_body[p][root_idx][1] = r[1];
        s_body[p][root_idx][2] = r[2];
    }
    __syncthreads();

    if (P > 0) {
        const int nphase = (root_idx == 2) ? 4 : NL;
        for (int phase = 0; phase < nphase; phase++) {
            const int i = (root_idx == 2) ? c_phase_limb[phase][warp] : (warp == 0 ? c_serial_limb[phase] : -1);
            if (i >= 0) {
                int src, dst;
                bool flip = false;
                if (root_idx == 2 && i == 1) {  // association.cpp:171-174
                    src = c_joint_pairs[2 * i + 1];
                    dst = c_joint_pairs[2 * i];
                    flip = true;
                } else {
                    src = c_joint_pairs[2 * i];
                    dst = c_joint_pairs[2 * i + 1];
                }
                const float* dstPeaks = pk + (size_t)dst * (MAXP + 1) * 3;
                const int dstSize = (int)dstPeaks[0];
                if (dstSize > 0) {
                    const float* sc = sc_img + (size_t)i * MAXP * MAXP;
                    unsigned char* used = s_used[warp];
                    for (int k = lane; k < dstSize; k += 32) used[k] = 0;
                    // candidate coordinates in registers: lane holds k2 = lane + 32*q
                    float cx[4], cy[4];
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const int k2 = lane + 32 * q;
                        cx[q] = (k2 < dstSize) ? dstPeaks[3 * (k2 + 1)] : 0.f;
                        cy[q] = (k2 < dstSize) ? dstPeaks[3 * (k2 + 1) + 1] : 0.f;
                    }
                    __syncwarp();
                    const float bl = c_bone_length[i];
                    // Score rows are prefetched one person ahead: the row index (remap of the source joint) and the
                    // source scores are fixed for the whole limb, only `used` changes from person to person.
                    auto load_row = [&](int k1, float(&row)[4]) {
                        const int rs = s_remap[src][k1];
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            const int k2 = lane + 32 * q;
                            row[q] = (k2 < dstSize) ? (flip ? sc[k2 * MAXP + rs] : sc[rs * MAXP + k2]) : -1.f;
                        }
                    };
                    auto next_valid = [&](int k1) {
                        while (k1 < P && (double)s_body[k1][src][2] < 1e-5) k1++;  // association.cpp:190
                        return k1;
                    };
                    int k1 = next_valid(0);
                    float cur[4], nxt[4];
                    if (k1 < P) load_row(k1, cur);
                    while (k1 < P) {
                        const int k1n = next_valid(k1 + 1);
                        if (k1n < P) load_row(k1n, nxt);
                        const float sx = s_body[k1][src][0], sy = s_body[k1][src][1];
                        const float bone_dist =
                            __double2float_rn(__ddiv_rn(__dmul_rn(1.2, (double)bl), (double)s_sorted[k1]));
                        float best = 0.0f;
                        int bestIdx = 0x7fffffff;
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            const int k2 = lane + 32 * q;
                            if (k2 < dstSize && !used[k2]) {
                                float score = cur[q];
                                if (dist_flag && score > 0) {
                                    const float ddx = __fsub_rn(sx, cx[q]), ddy = __fsub_rn(sy, cy[q]);
                                    const double d2 = __dadd_rn(__dmul_rn((double)ddx, (double)ddx),
                                                                __dmul_rn((double)ddy, (double)ddy));
                                    const float limb_dist = __double2float_rn(__dsqrt_rn(d2));
                                    const float t =
                                        __fsub_rn(__fdiv_rn(__fdiv_rn(bone_dist, limb_dist), 4.0f), 1.0f);
                                    score = __fadd_rn(score, (0.0f < t) ? 0.0f : t);  // std::min(t, 0.0f)
                                }
                                if (score > best) {  // ascending k2 within the lane: strict > keeps the first
                                    best = score;
                                    bestIdx = k2;
                                }
                            }
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) {
                            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                            const int oi = __shfl_xor_sync(0xffffffffu, bestIdx, o);
                            if (ob > best || (ob == best && oi < bestIdx)) {
                                best = ob;
                                bestIdx = oi;
                            }
                        }
                        if (best > 0) {  // association.cpp:220-228
                            if (lane == 0) {
                                s_body[k1][dst][0] = dstPeaks[3 * (bestIdx + 1)];
                                s_body[k1][dst][1] = dstPeaks[3 * (bestIdx + 1) + 1];
                                s_body[k1][dst][2] = dstPeaks[3 * (bestIdx + 1) + 2];
                                s_remap[dst][k1] = (unsigned char)bestIdx;
                                used[bestIdx] = 1;
                            }
                            __syncwarp();
                        }
                        k1 = k1n;
#pragma unroll
                        for (int q = 0; q < 4; q++) cur[q] = nxt[q];
                    }
                }
            }
            __syncthreads();
        }
    }
    // bodies [MAXP][NJ][4] = (x, y, 0, score); rows >= P zeroed
    for (int i = tid; i < MAXP * NJ; i += nthr) {
        const int p = i / NJ, j = i - p * NJ;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < P) v = make_float4(s_body[p][j][0], s_body[p][j][1], 0.f, s_body[p][j][2]);
        reinterpret_cast<float4*>(outb)[i] = v;
    }
}

// ---------------------------------------------------------------------------------------------
// 3D lift (rows C1-C4).  One CTA per image; a thread per (person, limb) for the relative-depth line
// statistics, then a thread per person for the bone chain + back-projection.  float32/float64 islands
// follow what the reference's numpy code does (see oracle/lift_numpy.py).
// ---------------------------------------------------------------------------------------------
constexpr int LIFT_THREADS = 256;

// numpy.linspace(start, stop, 10) in the dtype of its inputs: y = i*step + start (two roundings), last = stop
__device__ __forceinline__ float np_linspace10(float start, float stop, int i) {
    if (i == 9) return stop;
    const float delta = __fsub_rn(stop, start);
    const float step = __fdiv_rn(delta, 9.f);
    float y;
    if (step == 0.f)
        y = __fmul_rn(__fdiv_rn((float)i, 9.f), delta);
    else
        y = __fmul_rn((float)i, step);
    return __fadd_rn(y, start);
}
__device__ __forceinline__ double np_linspace10(double start, double stop, int i) {
    if (i == 9) return stop;
    const double delta = __dsub_rn(stop, start);
    const double step = __ddiv_rn(delta, 9.0);
    double y;
    if (step == 0.0)
        y = __dmul_rn(__ddiv_rn((double)i, 9.0), delta);
    else
        y = __dmul_rn((double)i, step);
    return __dadd_rn(y, start);
}
// a float64 intermediate stored into a column of the body array (float32 rounds, float64 keeps)
__device__ __forceinline__ void store_col(float& dst, double v) { dst = __double2float_rn(v); }
__device__ __forceinline__ void store_col(double& dst, double v) { dst = v; }
__device__ __forceinline__ int rint_to_int(float v) { return (int)rintf(v); }
__device__ __forceinline__ int rint_to_int(double v) { return (int)rint(v); }

// T = float : register_pred without ground truth (test_util.py:41) - float32 body rows, the run_inference mode.
// T = double: register_pred WITH ground truth (test_util.py:21-39) - rows follow the GT order and are float64
//             (np.zeros(..., np.float), test_util.py:35), so every float32 rounding of the other branch disappears.
template <typename T>
__global__ void __launch_bounds__(LIFT_THREADS, 1)
lift_kernel(const float* __restrict__ bodies, const int* __restrict__ counts, const float* __restrict__ det_d,
            const float* __restrict__ root_d, const double* __restrict__ scales, int h, int w, int root_n,
            T* __restrict__ pred2d_base, double* __restrict__ pred3d_base, double* __restrict__ root_depth_base,
            int* __restrict__ counts_out, long long s2d, long long s3d, long long srd, long long scnt,
            const double* __restrict__ gt_roots, const int* __restrict__ gt_counts, int gmax, double* __restrict__ dist_ws) {
    extern __shared__ __align__(16) unsigned char lift_smem[];
    typedef T BodyRow[NJ][4];
    BodyRow* s_b = reinterpret_cast<BodyRow*>(lift_smem);                                   // [MAXP][NJ][4]
    double(*s_dz)[NL] = reinterpret_cast<double(*)[NL]>(lift_smem + sizeof(T) * MAXP * NJ * 4);  // [MAXP][NL]
    int* s_keep = reinterpret_cast<int*>(lift_smem + sizeof(T) * MAXP * NJ * 4 + sizeof(double) * MAXP * NL);  // [MAXP]
    __shared__ int s_np;
    __shared__ double s_red_v[LIFT_THREADS / 32];
    __shared__ int s_red_i[LIFT_THREADS / 32];
    __shared__ unsigned char s_occ[MAXP];
    const int img = blockIdx.x, tid = threadIdx.x;
    const int hw = h * w;
    // per-image output slices (strides in elements: natural layout or smapb_record fields)
    T* pred2d = pred2d_base + (size_t)img * s2d;
    double* pred3d = pred3d_base + (size_t)img * s3d;
    double* root_depth = root_depth_base + (size_t)img * srd;
    const int P = counts[img];
    const float* b = bodies + (size_t)img * MAXP * NJ * 4;
    const float* dd = det_d + (size_t)img * NL * hw;
    const float* rd = root_d + (size_t)img * hw;
    const double* sc = scales + (size_t)img * 9;  // scale, img_w, img_h, net_w, net_h, fx, fy, cx, cy
    if (gt_roots == nullptr) {
        if (tid == 0) {  // register_pred without GT (test_util.py:41): keep persons whose root score != 0
            int n = 0;
            for (int p = 0; p < P; p++)
                if (b[(p * NJ + root_n) * 4 + 3] != 0.f) s_keep[n++] = p;
            s_np = n;
        }
        __syncthreads();
    } else {
        // register_pred with GT (test_util.py:21-39): distance matrix of GT roots x predicted roots, then the entries
        // below 30 px are visited in ascending (distance, row-major index) order - the reference takes the minimum, walks
        // all entries equal to it in np.where order, overwrites them with 50 and repeats - and a pair is made when both
        // its GT person and its prediction are still free.
        const int G = min(gt_counts[img], min(gmax, MAXP));
        const bool skip = (P == 0) || (G <= 0);  // no prediction: empty result (:19-20); no GT person: frame skipped (test.py:83-84)
        double* D = dist_ws + (size_t)img * MAXP * MAXP;
        const double* gr = gt_roots + (size_t)img * gmax * 2;
        if (!skip) {
            for (int i = tid; i < G * P; i += LIFT_THREADS) {
                const int g = i / P, p = i - g * P;
                const float px = __fmul_rn(b[(p * NJ + root_n) * 4 + 0], 4.f), py = __fmul_rn(b[(p * NJ + root_n) * 4 + 1], 4.f);
                const double dx = __dsub_rn(gr[2 * g], (double)px), dy = __dsub_rn(gr[2 * g + 1], (double)py);
                D[i] = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));  // np.linalg.norm(axis=2)
            }
            for (int g = tid; g < G; g += LIFT_THREADS) s_keep[g] = -1;
            for (int p = tid; p < P; p += LIFT_THREADS) s_occ[p] = 0;
        }
        __syncthreads();
        while (!skip) {
            double bv = 1e300;
            int bi = 0x7fffffff;
            for (int i = tid; i < G * P; i += LIFT_THREADS) {
                const double v = D[i];
                if (v < 30.0 && (v < bv || (v == bv && i < bi))) bv = v, bi = i;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov < bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
            }
            if ((tid & 31) == 0) s_red_v[tid >> 5] = bv, s_red_i[tid >> 5] = bi;
            __syncthreads();
            bv = s_red_v[0], bi = s_red_i[0];
            for (int k = 1; k < LIFT_THREADS / 32; k++)
                if (s_red_v[k] < bv || (s_red_v[k] == bv && s_red_i[k] < bi)) bv = s_red_v[k], bi = s_red_i[k];
            if (bi == 0x7fffffff) break;  // uniform: np.min(distance_array) >= 30
            if (tid == 0) {
                const int g = bi / P, p = bi - g * P;
                D[bi] = 50.0;
                if (s_keep[g] < 0 && !s_occ[p]) s_keep[g] = p, s_occ[p] = 1;
            }
            __syncthreads();  // D / s_keep / s_occ updates visible; s_red reusable
        }
        if (tid == 0) s_np = skip ? 0 : G;
        __syncthreads();
    }
    const int NP = s_np;
    for (int i = tid; i < NP * NJ; i += LIFT_THREADS) {
        const int p = i / NJ, j = i - p * NJ;
        if (s_keep[p] < 0) {  // unmatched GT person: zero row (test_util.py:35)
            s_b[p][j][0] = s_b[p][j][1] = s_b[p][j][2] = s_b[p][j][3] = (T)0;
            continue;
        }
        const float* s = b + (s_keep[p] * NJ + j) * 4;
        s_b[p][j][0] = (T)__fmul_rn(s[0], 4.f);  // test.py:117 (float32 tensor op, then widened in the GT branch)
        s_b[p][j][1] = (T)__fmul_rn(s[1], 4.f);
        s_b[p][j][2] = (T)s[2];
        s_b[p][j][3] = (T)s[3];
    }
    __syncthreads();
    // numpy percentile constants (method 'linear'): virtual index (n-1)*q, gamma = frac
    const double vi10 = 9.0 * (10.0 / 100.0), vi90 = 9.0 * (90.0 / 100.0);
    const double g10 = vi10 - floor(vi10), g90 = vi90 - floor(vi90);
    const int i10 = (int)floor(vi10), i90 = (int)floor(vi90);
    for (int i = tid; i < NP * NL; i += LIFT_THREADS) {
        const int p = i / NL, k = i - p * NL;
        const int ja = c_joint_pairs[2 * k], jb = c_joint_pairs[2 * k + 1];
        double dz = 0.0;
        if (s_b[p][root_n][3] > 0 && s_b[p][jb][3] > 0 && s_b[p][ja][3] > 0) {
            float v[10];
#pragma unroll
            for (int t = 0; t < 10; t++) {
                const int xx = rint_to_int(np_linspace10(s_b[p][ja][0], s_b[p][jb][0], t));
                const int yy = rint_to_int(np_linspace10(s_b[p][ja][1], s_b[p][jb][1], t));
                const int hx = min(w - 1, max(0, xx >> 2)), hy = min(h - 1, max(0, yy >> 2));
                v[t] = dd[(size_t)k * hw + hy * w + hx];
            }
            float s[10];
#pragma unroll
            for (int t = 0; t < 10; t++) s[t] = v[t];
#pragma unroll
            for (int a = 1; a < 10; a++) {  // insertion sort
                const float key = s[a];
                int q = a - 1;
                while (q >= 0 && s[q] > key) {
                    s[q + 1] = s[q];
                    q--;
                }
                s[q + 1] = key;
            }
            // numpy _lerp: a + (b-a)*t, or b - (b-a)*(1-t) where t >= 0.5; (b-a) in float32
            auto lerp = [](float a, float bb, double t) {
                const double diff = (double)__fsub_rn(bb, a);
                return (t >= 0.5) ? __dsub_rn((double)bb, __dmul_rn(diff, __dsub_rn(1.0, t)))
                                  : __dadd_rn((double)a, __dmul_rn(diff, t));
            };
            const double lo = lerp(s[i10], s[i10 + 1], g10);
            const double hi = lerp(s[i90], s[i90 + 1], g90);
            const float flo = __double2float_rn(lo), fhi = __double2float_rn(hi);
#pragma unroll
            for (int t = 0; t < 10; t++) {
                if ((double)v[t] < lo) v[t] = flo;
                if ((double)v[t] > hi) v[t] = fhi;
            }
            // numpy float32 pairwise sum for n = 10: 8-way unrolled block + 2 tail adds
            const float r = __fadd_rn(__fadd_rn(__fadd_rn(v[0], v[1]), __fadd_rn(v[2], v[3])),
                                      __fadd_rn(__fadd_rn(v[4], v[5]), __fadd_rn(v[6], v[7])));
            const float tot = __fadd_rn(__fadd_rn(r, v[8]), v[9]);
            dz = (double)__fdiv_rn(tot, 10.f);
        }
        s_dz[p][k] = dz;
    }
    __syncthreads();
    for (int p = tid; p < NP; p += LIFT_THREADS) {
        double rdep = 0.0;
        if (s_b[p][root_n][3] > 0) {
            const int ry = (int)s_b[p][root_n][1], rx = (int)s_b[p][root_n][0];
            const float r = rd[min(h - 1, max(0, ry >> 2)) * w + min(w - 1, max(0, rx >> 2))];
            rdep = __dmul_rn(__dmul_rn((double)r, sc[0]), sc[5]);  // test_util.py:66
            // chain_bones (test_util.py:45-57): column written in place (float32 rows round, float64 rows do not)
            s_b[p][2][2] = (T)0;
            store_col(s_b[p][0][2], __dsub_rn((double)s_b[p][2][2], s_dz[p][1]));
            store_col(s_b[p][1][2], __dadd_rn((double)s_b[p][0][2], s_dz[p][0]));
            for (int k = 2; k < NL; k++) {
                const int ja = c_joint_pairs[2 * k], jb = c_joint_pairs[2 * k + 1];
                store_col(s_b[p][jb][2], __dadd_rn((double)s_b[p][ja][2], s_dz[p][k]));
            }
        }
        root_depth[p] = rdep;
        // gen_3d_pose (test_util.py:89-99) + get_3d_points/back_projection (post_3d.py:4-27)
        const double s = sc[0];
        const double offx = __ddiv_rn(__dsub_rn(__ddiv_rn(sc[3], s), sc[1]), 2.0);
        const double offy = __ddiv_rn(__dsub_rn(__ddiv_rn(sc[4], s), sc[2]), 2.0);
        const bool has_root = s_b[p][root_n][3] != (T)0;
        for (int j = 0; j < NJ; j++) {
            T* o2 = pred2d + ((size_t)p * NJ + j) * 4;
            o2[0] = s_b[p][j][0];
            o2[1] = s_b[p][j][1];
            o2[2] = s_b[p][j][2];
            o2[3] = s_b[p][j][3];
            double* o3 = pred3d + ((size_t)p * NJ + j) * 4;
            double X = 0, Y = 0, Z = 0;
            const T score = s_b[p][j][3];
            if (has_root && score != (T)0) {
                T bx, by, bz;
                store_col(bx, __dsub_rn(__ddiv_rn((double)s_b[p][j][0], s), offx));
                store_col(by, __dsub_rn(__ddiv_rn((double)s_b[p][j][1], s), offy));
                store_col(bz, __dadd_rn((double)s_b[p][j][2], rdep));
                const double d = (double)bz;
                X = __ddiv_rn(__dmul_rn(__dsub_rn((double)bx, sc[7]), d), sc[5]);
                Y = __ddiv_rn(__dmul_rn(__dsub_rn((double)by, sc[8]), d), sc[6]);
                Z = d;
            }
            o3[0] = X;
            o3[1] = Y;
            o3[2] = Z;
            o3[3] = (double)score;
        }
    }
    // zero the unused tail of the fixed-stride record (all-gather payload must be deterministic)
    for (int i = NP * NJ * 4 + tid; i < MAXP * NJ * 4; i += LIFT_THREADS) {
        pred2d[i] = (T)0;
        pred3d[i] = 0.0;
    }
    for (int i = NP + tid; i < MAXP; i += LIFT_THREADS) root_depth[i] = 0.0;
    if (tid == 0) {
        counts_out[(size_t)img * scnt] = NP;
        if (scnt > 1) counts_out[(size_t)img * scnt + 1] = 0;  // smapb_record::pad_
    }
}

// ---------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------
static size_t paf_pk_bytes() { return 16 + 4 * (MAXP + 1) * 4; }
static size_t paf_smem(int h, int w) { return paf_pk_bytes() + (size_t)h * w * 8; }
static bool paf_staged(int h, int w) { return paf_smem(h, w) <= 232448 && (h * w) % 2 == 0; }
// Any map size: NMS streams from global memory; PAF stages both planes in shared memory when they fit (w*h*8 + 2 KB
// <= 227 KB, needs h*w % 2 == 0 for the 16-byte bulk copies) and gathers from global memory / L2 otherwise.  The reference
// hard-codes 128 x 208 (extensions/association.cpp:21).
int assoc_configure(int h, int w, const char** err) {
    static const char* e_small = "association: heat-map must be at least 3 x 3";
    if (h < 3 || w < 3) {
        *err = e_small;
        return -1;
    }
    cudaError_t e = cudaSuccess;
    if (paf_staged(h, w))
        e = cudaFuncSetAttribute(paf_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)paf_smem(h, w));
    if (e != cudaSuccess) {
        *err = cudaGetErrorString(e);
        return -2;
    }
    return 0;
}

size_t nms_mask_words(int B, int h, int w) { return (size_t)B * NJ * ((h * w + 31) / 32); }

cudaError_t launch_nms(const float* hms, int nchan, int B, int h, int w, float thr, float* peaks, uint32_t* masks,
                       cudaStream_t st) {
    const long long words = (long long)nms_mask_words(B, h, w);
    const bool vec = (h * w) % 128 == 0;
    const long long warps_needed = vec ? (words + 15) / 16 : words;  // 16 words (VEC, 4 groups) or 1 word per warp step
    long long blocks = (warps_needed * 32 + NMSF_THREADS - 1) / NMSF_THREADS;
    const long long cap = vec ? 132LL * 4 : 132LL * 8 * 4;  // VEC: one persistent wave; scalar: the warps stride over the rest
    if (blocks > cap) blocks = cap;
    if (vec)
        nms_flag_kernel<true><<<(unsigned)blocks, NMSF_THREADS, 0, st>>>(hms, nchan, B, h, w, thr, masks);
    else
        nms_flag_kernel<false><<<(unsigned)blocks, NMSF_THREADS, 0, st>>>(hms, nchan, B, h, w, thr, masks);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    nms_compact_kernel<<<dim3(NJ, B), NMSC_THREADS, 0, st>>>(hms, nchan, h, w, masks, peaks);
    return cudaGetLastError();
}
cudaError_t launch_paf(const float* hms, int nchan, int B, int h, int w, const float* peaks, float* scores,
                       int dense_fill, cudaStream_t st) {
    if (paf_staged(h, w))
        paf_kernel<true><<<dim3(NL, B), PAF_THREADS, paf_smem(h, w), st>>>(hms, nchan, h, w, peaks, scores, dense_fill);
    else
        paf_kernel<false><<<dim3(NL, B), PAF_THREADS, paf_pk_bytes(), st>>>(hms, nchan, h, w, peaks, scores, dense_fill);
    return cudaGetLastError();
}
cudaError_t launch_group(const float* peaks, const float* scores, const float* rdepth, int B, int h, int w,
                         int root_idx, int dist_flag, float* bodies, int* counts, cudaStream_t st) {
    group_kernel<<<B, GROUP_WARPS * 32, 0, st>>>(peaks, scores, rdepth, h, w, root_idx, dist_flag, bodies, counts);
    return cudaGetLastError();
}
template <typename T>
static size_t lift_smem() { return sizeof(T) * MAXP * NJ * 4 + sizeof(double) * MAXP * NL + sizeof(int) * MAXP; }

cudaError_t launch_lift(const float* bodies, const int* counts, const float* det_d, const float* root_d,
                        const double* scales, int B, int h, int w, int root_n, float* pred2d, double* pred3d,
                        double* root_depth, int* counts_out, long long s2d, long long s3d, long long srd, long long scnt,
                        cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(lift_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lift_smem<float>());
        if (e != cudaSuccess) return e;
        configured = true;
    }
    lift_kernel<float><<<B, LIFT_THREADS, lift_smem<float>(), st>>>(bodies, counts, det_d, root_d, scales, h, w, root_n, pred2d,
                                                                   pred3d, root_depth, counts_out, s2d, s3d, srd, scnt, nullptr,
                                                                   nullptr, 0, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_lift_gt(const float* bodies, const int* counts, const float* det_d, const float* root_d,
                           const double* scales, const double* gt_roots, const int* gt_counts, int gmax, double* dist_ws, int B,
                           int h, int w, int root_n, double* pred2d, double* pred3d, double* root_depth, int* counts_out,
                           cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(lift_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lift_smem<double>());
        if (e != cudaSuccess) return e;
        configured = true;
    }
    lift_kernel<double><<<B, LIFT_THREADS, lift_smem<double>(), st>>>(bodies, counts, det_d, root_d, scales, h, w, root_n, pred2d,
                                                                     pred3d, root_depth, counts_out, (long long)MAXP * NJ * 4,
                                                                     (long long)MAXP * NJ * 4, MAXP, 1, gt_roots, gt_counts, gmax,
                                                                     dist_ws);
    return cudaGetLastError();
}

}  // namespace smapb
