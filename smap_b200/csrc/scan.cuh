// The batch-wide exclusive scan of the image encoders (jpeg_enc.cu, png_enc.cu): uint32 counts -> uint64 offsets, the
// grand total after the last.  Three launches whatever n: per-tile sums, one CTA scans the tile sums, per-tile apply.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>

#include "decode_host.h"

namespace smapb {
namespace {

constexpr int SCAN_THREADS = 1024, SCAN_ITEMS = 4, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// CTA-wide exclusive sum of one value per thread (blockDim.x == SCAN_THREADS); *total = the CTA's sum
__device__ __forceinline__ unsigned long long block_exclusive(unsigned long long v, unsigned long long* total) {
    __shared__ unsigned long long warp_sums[SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned long long s = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    const unsigned long long before = (wid ? warp_sums[wid - 1] : 0) + x - v;
    *total = warp_sums[SCAN_THREADS / 32 - 1];
    __syncthreads();
    return before;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_reduce_kernel(const uint32_t* __restrict__ in, long long n,
                                                                   unsigned long long* __restrict__ tile_sums) {
    const long long base = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    unsigned long long s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; i++)
        if (base + i < n) s += in[base + i];
    unsigned long long total;
    block_exclusive(s, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_tiles_kernel(unsigned long long* __restrict__ tile_sums, long long ntiles,
                                                                  unsigned long long* __restrict__ grand) {
    unsigned long long carry = 0;
    for (long long b = 0; b < ntiles; b += SCAN_THREADS) {
        const long long i = b + threadIdx.x;
        const unsigned long long v = i < ntiles ? tile_sums[i] : 0;
        unsigned long long total;
        const unsigned long long ex = block_exclusive(v, &total);
        if (i < ntiles) tile_sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *grand = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(const uint32_t* __restrict__ in, long long n,
                                                                  const unsigned long long* __restrict__ tile_sums,
                                                                  unsigned long long* __restrict__ out) {
    const long long base = (long long)blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    unsigned long long s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; i++) {
        v[i] = base + i < n ? in[base + i] : 0;
        s += v[i];
    }
    unsigned long long total;
    unsigned long long run = tile_sums[blockIdx.x] + block_exclusive(s, &total);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; i++) {
        if (base + i < n) out[base + i] = run;
        run += v[i];
    }
}

// exclusive scan of in[0..n) into out[0..n], out[n] = the sum; 3 launches; tiles is the scan's scratch
inline int exclusive_scan(DeviceBuffer<unsigned long long>* tiles, const uint32_t* in, long long n, unsigned long long* out,
                          cudaStream_t st, std::string* err) {
    const long long nt = std::max(1ll, (n + SCAN_TILE - 1) / SCAN_TILE);
    DECODE_CK(tiles->grow((size_t)nt));
    scan_reduce_kernel<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(in, n, *tiles);
    scan_tiles_kernel<<<1, SCAN_THREADS, 0, st>>>(*tiles, nt, out + n);
    scan_apply_kernel<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(in, n, *tiles, out);
    DECODE_CK(cudaGetLastError());
    return 0;
}

}  // namespace
}  // namespace smapb
