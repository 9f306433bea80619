// Baseline JPEG encoding on the GPU, byte-identical to cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, q]) (libjpeg-turbo
// defaults: 4:2:0, standard Huffman tables, no restart interval), restated on the CPU by oracle/jpeg_encode_numpy.py.
//
// One launch per phase for the whole batch (frames of any sizes):
//   overlay   (records only) the composite stage's label planes (overlay.cu, view3d.cu);
//   colour    one thread per chroma sample: its 2x2 pixels (labelled ones replaced by their element's colour), fixed-point
//             RGB -> YCbCr, the four luma samples and the biased 2x2 chroma means, edge-replicated to the MCU grid;
//   fdct      one thread per block: level shift, accurate-integer FDCT, quantisation, zigzag int16 coefficients; luma
//             blocks past the frame's block grid are libjpeg's dummy blocks (zero AC, the DC of the block before);
//   bits      one thread per block: the DC difference and the run/size tokens, summed in bits;
//   scan      exclusive scan of the bit counts over the batch (three launches) -> each block's bit offset;
//   zero      each block clears the words whose first bit it owns;
//   pack      each block writes its tokens MSB-first at its offset; the words it shares with its neighbours are merged
//             with atomicOr, so the result does not depend on the order; the last block pads its byte with 1-bits;
//   ff        each block counts the 0xFF bytes whose first bit it owns; scanned like the bits (three launches);
//   totals    per image: stuffed size and output offset (one D2H and a synchronisation bring them to the host);
//   scatter   each block copies its bytes, a 0x00 after every 0xFF, into the output, which one D2H brings back.
// The headers are written by the host from the quality and the frame size.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "decode_host.h"
#include "jpeg_enc.h"
#include "overlay.cuh"
#include "scan.cuh"

namespace smapb {

namespace {

constexpr int BLOCK_BITS_MAX = 22 + 63 * 26;  // the longest DC token + 63 tokens of run 0 / size 10 (jpeg_encode_numpy)

const int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// ITU-T T.81 Annex K.1 quantisation tables in zigzag order, K.3 Huffman tables
const uint8_t kBaseQ[2][64] = {
    {16, 11, 12, 14, 12, 10, 16, 14, 13, 14, 18, 17, 16, 19, 24, 40, 26, 24, 22, 22, 24, 49,
     35, 37, 29, 40, 58, 51, 61, 60, 57, 51, 56, 55, 64, 72, 92, 78, 64, 68, 87, 69, 55, 56,
     80, 109, 81, 87, 95, 98, 103, 104, 103, 62, 77, 113, 121, 112, 100, 120, 92, 101, 103, 99},
    {17, 18, 18, 24, 21, 24, 47, 26, 26, 47, 99, 66, 56, 66, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
const uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
const uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
const uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// quantisers and Huffman codes of one call, uploaded with the image descriptors
struct EncTables {
    uint16_t qdiv[2][64];  // 8 * Q (the FDCT's output scale), natural order
    uint16_t dc_code[2][12];
    uint8_t dc_len[2][12];
    uint16_t ac_code[2][256];
    uint8_t ac_len[2][256];
};

struct EncImg {
    int h, w, mx, my, bw, bh;  // the encoded image's size (its Composite's), MCU columns / rows, luma block columns / rows
    long long blk0;  // first block in the batch's block order
    long long plane0;  // Y plane [16 my][16 mx], then Cb and Cr [8 my][8 mx]
    long long word0;  // first word of the image's bit buffer
    long long bound_bits;  // blocks * BLOCK_BITS_MAX
};

// per-image results of the totals kernel
struct EncTotals {
    long long bits, stuffed, out0;
};

__device__ __forceinline__ int find_image(const EncImg* im, int n, long long g) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (im[mid].blk0 <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// libjpeg-turbo's RGB -> YCbCr: 16-bit fixed point, Cb and Cr rounded with 1/2 - epsilon
__device__ __forceinline__ int ycc_y(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int ycc_cb(int r, int g, int b) { return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16; }
__device__ __forceinline__ int ycc_cr(int r, int g, int b) { return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16; }

__global__ void __launch_bounds__(256) colour_kernel(const EncImg* __restrict__ imgs, const Composite* __restrict__ comps,
                                                     const int* __restrict__ labels, uint8_t* __restrict__ planes) {
    const EncImg& I = imgs[blockIdx.y];
    const Composite& P = comps[blockIdx.y];
    const int cw = 8 * I.mx;
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)cw * 8 * I.my) return;
    const int cx = (int)(k % cw), cy = (int)(k / cw);
    uint8_t* Y = planes + I.plane0;
    const int yw = 16 * I.mx;
    // luma: the frame with its last column and row replicated
    int cb = 0, cr = 0;
    const int ch = (I.h + 1) >> 1;
    const int cys = min(cy, ch - 1);  // chroma rows past the frame's replicate its last chroma row
#pragma unroll
    for (int dy = 0; dy < 2; dy++) {
#pragma unroll
        for (int dx = 0; dx < 2; dx++) {
            const int x = min(2 * cx + dx, I.w - 1);
            int b, g, r;
            load_pixel(P, labels, x, min(2 * cy + dy, I.h - 1), &b, &g, &r);
            Y[(size_t)(2 * cy + dy) * yw + 2 * cx + dx] = (uint8_t)ycc_y(r, g, b);
            if (cys != cy) load_pixel(P, labels, x, min(2 * cys + dy, I.h - 1), &b, &g, &r);
            cb += ycc_cb(r, g, b);
            cr += ycc_cr(r, g, b);
        }
    }
    const int bias = 1 + (cx & 1);
    const size_t c = (size_t)cy * cw + cx, csize = (size_t)64 * I.mx * I.my;
    uint8_t* C = Y + 4 * csize;
    C[c] = (uint8_t)((cb + bias) >> 2);
    C[csize + c] = (uint8_t)((cr + bias) >> 2);
}

// ---- forward DCT and quantisation -------------------------------------------------------------------------------
#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

// one pass of the islow FDCT over 8 values with stride s; first: pass 1 (rows), else pass 2 (columns)
template <bool first>
__device__ __forceinline__ void fdct8(int* d, int s) {
    constexpr int CB = 13, P1 = 2, SH = first ? CB - P1 : CB + P1;
    const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
    const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    if (first) {
        d[0] = (t10 + t11) * 4;
        d[4 * s] = (t10 - t11) * 4;
    } else {
        d[0] = DESCALE(t10 + t11, P1);
        d[4 * s] = DESCALE(t10 - t11, P1);
    }
    int z1 = (t12 + t13) * 4433;
    d[2 * s] = DESCALE(z1 + t13 * 6270, SH);
    d[6 * s] = DESCALE(z1 - t12 * 15137, SH);
    z1 = t4 + t7;
    int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
    const int z5 = (z3 + z4) * 9633;
    z1 *= -7373, z2 *= -20995;
    z3 = z3 * -16069 + z5, z4 = z4 * -3196 + z5;
    d[7 * s] = DESCALE(t4 * 2446 + z1 + z3, SH);
    d[5 * s] = DESCALE(t5 * 16819 + z2 + z4, SH);
    d[3 * s] = DESCALE(t6 * 25172 + z2 + z3, SH);
    d[s] = DESCALE(t7 * 12299 + z1 + z4, SH);
}

// zigzag position of natural index i (the inverse of kZigzag); a constant once the loops are unrolled
__device__ __forceinline__ constexpr int zigzag_pos(int i) {
    constexpr int pos[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                             41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                             46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
    return pos[i];
}

__device__ __forceinline__ int quant(int v, int div) {
    const int a = ((v < 0 ? -v : v) + (div >> 1)) / div;
    return v < 0 ? -a : a;
}

// the block's 64 samples: component k of MCU (mcx, mcy) (0..3 luma 2x2, 4 Cb, 5 Cr), luma sub-block (sx, sy)
__device__ __forceinline__ const uint8_t* block_src(const EncImg& I, const uint8_t* planes, int k, int mcx, int mcy, int* stride) {
    const uint8_t* Y = planes + I.plane0;
    if (k < 4) {
        *stride = 16 * I.mx;
        return Y + (size_t)(16 * mcy + 8 * (k >> 1)) * *stride + 16 * mcx + 8 * (k & 1);
    }
    *stride = 8 * I.mx;
    return Y + (size_t)256 * I.mx * I.my + (size_t)(k - 4) * 64 * I.mx * I.my + (size_t)(8 * mcy) * *stride + 8 * mcx;
}

__device__ __forceinline__ bool luma_real(const EncImg& I, int k, int mcx, int mcy) {
    return 2 * mcx + (k & 1) < I.bw && 2 * mcy + (k >> 1) < I.bh;
}

__global__ void __launch_bounds__(128) fdct_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                   const EncTables* __restrict__ tab, const uint8_t* __restrict__ planes,
                                                   int16_t* __restrict__ coef) {
    __shared__ uint16_t qdiv[2][64];
    for (int i = threadIdx.x; i < 128; i += blockDim.x) qdiv[i >> 6][i & 63] = tab->qdiv[i >> 6][i & 63];
    __syncthreads();
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const EncImg& I = imgs[find_image(imgs, n, g)];
    const long long local = g - I.blk0;
    const int k = (int)(local % 6);
    const long long mcu = local / 6;
    const int mcx = (int)(mcu % I.mx), mcy = (int)(mcu / I.mx);
    const int t = k < 4 ? 0 : 1;
    int16_t* out = coef + g * 64;
    int stride;
    if (k < 4 && !luma_real(I, k, mcx, mcy)) {
        // dummy block: zero AC, the DC of the last real block before it in the MCU (block 0 always is); a DC is the
        // plain sum of the level-shifted samples
        int j = k - 1;
        while (!luma_real(I, j, mcx, mcy)) j--;
        const uint8_t* s = block_src(I, planes, j, mcx, mcy, &stride);
        int sum = 0;
        for (int y = 0; y < 8; y++)
            for (int x = 0; x < 8; x++) sum += s[(size_t)y * stride + x];
        uint4* o = reinterpret_cast<uint4*>(out);
#pragma unroll
        for (int i = 0; i < 8; i++) o[i] = make_uint4(0, 0, 0, 0);
        out[0] = (int16_t)quant(sum - 64 * 128, qdiv[0][0]);
        return;
    }
    const uint8_t* s = block_src(I, planes, k, mcx, mcy, &stride);
    int d[64];
#pragma unroll
    for (int y = 0; y < 8; y++) {
        const uint2 v = *reinterpret_cast<const uint2*>(s + (size_t)y * stride);
#pragma unroll
        for (int x = 0; x < 4; x++) {
            d[y * 8 + x] = (int)((v.x >> (8 * x)) & 255) - 128;
            d[y * 8 + 4 + x] = (int)((v.y >> (8 * x)) & 255) - 128;
        }
    }
#pragma unroll
    for (int y = 0; y < 8; y++) fdct8<true>(d + 8 * y, 1);
#pragma unroll
    for (int x = 0; x < 8; x++) fdct8<false>(d + x, 8);
    // quantise in natural order, store in zigzag order: 32 packed pairs
    uint32_t packed[32];
#pragma unroll
    for (int i = 0; i < 32; i++) packed[i] = 0;
#pragma unroll
    for (int i = 0; i < 64; i++) {
        const int z = zigzag_pos(i);
        packed[z >> 1] |= (uint32_t)(uint16_t)(int16_t)quant(d[i], qdiv[t][i]) << (16 * (z & 1));
    }
    uint4* o = reinterpret_cast<uint4*>(out);
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = make_uint4(packed[4 * i], packed[4 * i + 1], packed[4 * i + 2], packed[4 * i + 3]);
}

// ---- entropy coding -----------------------------------------------------------------------------------------------
__device__ __forceinline__ int category(int v) { return v == 0 ? 0 : 32 - __clz(v < 0 ? -v : v); }
__device__ __forceinline__ uint32_t extra_bits(int v, int s) { return (uint32_t)(v < 0 ? v + (1 << s) - 1 : v) & ((1u << s) - 1); }

// calls emit(bits, length) for every token of block g, in stream order (lengths <= 27)
template <typename Emit>
__device__ __forceinline__ void block_tokens(const EncImg& I, const EncTables& T, const int16_t* __restrict__ coef, long long g,
                                             Emit emit) {
    const long long local = g - I.blk0;
    const int k = (int)(local % 6);
    const int t = k < 4 ? 0 : 1;
    long long prev = -1;  // the previous block of the same component in scan order
    if (k == 1 || k == 2 || k == 3) prev = g - 1;
    else if (local >= 6) prev = k == 0 ? g - 3 : g - 6;
    const int4* c4 = reinterpret_cast<const int4*>(coef + g * 64);
    uint32_t w[32];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int4 v = c4[i];
        w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
    }
    const int dc = (int16_t)(w[0] & 0xFFFF);
    const int diff = dc - (prev >= 0 ? (int)coef[prev * 64] : 0);
    int s = category(diff);
    emit(((uint32_t)T.dc_code[t][s] << s) | extra_bits(diff, s), T.dc_len[t][s] + s);
    uint64_t nz = 0;
#pragma unroll
    for (int i = 1; i < 64; i++)
        if ((w[i >> 1] >> (16 * (i & 1))) & 0xFFFF) nz |= 1ull << i;
    int last = 0;
    while (nz) {
        const int i = __ffsll((long long)nz) - 1;
        nz &= nz - 1;
        int run = i - last - 1;
        for (; run >= 16; run -= 16) emit(T.ac_code[t][0xF0], T.ac_len[t][0xF0]);
        const int v = coef[g * 64 + i];  // the line the block's loads just brought in
        s = category(v);
        const int sym = (run << 4) | s;
        emit(((uint32_t)T.ac_code[t][sym] << s) | extra_bits(v, s), T.ac_len[t][sym] + s);
        last = i;
    }
    if (last < 63) emit(T.ac_code[t][0], T.ac_len[t][0]);
}

__device__ __forceinline__ void load_tables(EncTables* sh, const EncTables* g) {
    const int nw = sizeof(EncTables) / 4;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) reinterpret_cast<uint32_t*>(sh)[i] = reinterpret_cast<const uint32_t*>(g)[i];
    __syncthreads();
}

__global__ void __launch_bounds__(128) bits_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                   const EncTables* __restrict__ tab, const int16_t* __restrict__ coef,
                                                   uint32_t* __restrict__ bits) {
    __shared__ EncTables T;
    load_tables(&T, tab);
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const EncImg& I = imgs[find_image(imgs, n, g)];
    uint32_t total = 0;
    block_tokens(I, T, coef, g, [&](uint32_t, int len) { total += len; });
    bits[g] = total;
}

// ---- packing and stuffing ------------------------------------------------------------------------------------------
// a block's bit range inside its image: [b0, b1); the last block's range ends at the image's total
struct BitRange {
    long long b0, b1;
    bool last;
};

__device__ __forceinline__ BitRange bit_range(const EncImg& I, const EncImg* next, long long nblk, long long g,
                                              const unsigned long long* __restrict__ off) {
    const long long end = next ? next->blk0 : nblk;
    BitRange r;
    r.b0 = (long long)(off[g] - off[I.blk0]);
    r.b1 = (long long)(off[g + 1] - off[I.blk0]);
    r.last = g + 1 == end;
    return r;
}

__global__ void __launch_bounds__(256) zero_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                   const unsigned long long* __restrict__ off, uint32_t* __restrict__ words) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const int i = find_image(imgs, n, g);
    const EncImg& I = imgs[i];
    const BitRange r = bit_range(I, i + 1 < n ? &imgs[i + 1] : nullptr, nblk, g, off);
    if (r.b1 > I.bound_bits) return;
    for (long long w = (r.b0 + 31) >> 5; 32 * w < r.b1; w++) words[I.word0 + w] = 0;  // the words whose first bit is ours
}

__global__ void __launch_bounds__(128) pack_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                   const EncTables* __restrict__ tab, const int16_t* __restrict__ coef,
                                                   const unsigned long long* __restrict__ off, uint32_t* __restrict__ words) {
    __shared__ EncTables T;
    load_tables(&T, tab);
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const int i = find_image(imgs, n, g);
    const EncImg& I = imgs[i];
    const BitRange r = bit_range(I, i + 1 < n ? &imgs[i + 1] : nullptr, nblk, g, off);
    if (r.b1 > I.bound_bits) return;
    uint32_t* W = words + I.word0;
    long long wi = r.b0 >> 5;
    int nacc = (int)(r.b0 & 31);
    unsigned long long acc = 0;
    bool shared_word = true;  // the first word may hold the previous block's bits
    auto emit = [&](uint32_t v, int len) {
        acc = (acc << len) | v;
        nacc += len;
        if (nacc >= 32) {
            const uint32_t word = (uint32_t)(acc >> (nacc - 32));
            nacc -= 32;
            if (shared_word) atomicOr(&W[wi], word);
            else W[wi] = word;
            shared_word = false;
            wi++;
        }
    };
    block_tokens(I, T, coef, g, emit);
    if (r.last && (r.b1 & 7)) emit((1u << (8 - (r.b1 & 7))) - 1, 8 - (int)(r.b1 & 7));  // 1-bits to the byte boundary
    if (nacc > 0) atomicOr(&W[wi], (uint32_t)(acc << (32 - nacc)));  // shared with the next block
}

__device__ __forceinline__ uint8_t stream_byte(const uint32_t* W, long long b) { return (uint8_t)(W[b >> 2] >> (24 - 8 * (b & 3))); }

// the bytes whose first bit lies in the block's range
__device__ __forceinline__ void owned_bytes(const BitRange& r, long long* first, long long* end) {
    *first = (r.b0 + 7) >> 3;
    *end = (r.b1 + 7) >> 3;
}

__global__ void __launch_bounds__(256) ff_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                 const unsigned long long* __restrict__ off, const uint32_t* __restrict__ words,
                                                 uint32_t* __restrict__ ff) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const int i = find_image(imgs, n, g);
    const EncImg& I = imgs[i];
    const BitRange r = bit_range(I, i + 1 < n ? &imgs[i + 1] : nullptr, nblk, g, off);
    uint32_t c = 0;
    if (r.b1 <= I.bound_bits) {
        long long b, e;
        owned_bytes(r, &b, &e);
        for (; b < e; b++) c += stream_byte(words + I.word0, b) == 0xFF;
    }
    ff[g] = c;
}

__global__ void totals_kernel(const EncImg* __restrict__ imgs, int n, long long nblk, const unsigned long long* __restrict__ off,
                              const unsigned long long* __restrict__ ffoff, long long header_bytes, EncTotals* __restrict__ tot) {
    long long out = 0;
    for (int i = 0; i < n; i++) {
        const long long b0 = imgs[i].blk0, b1 = i + 1 < n ? imgs[i + 1].blk0 : nblk;
        EncTotals t;
        t.bits = (long long)(off[b1] - off[b0]);
        t.stuffed = (t.bits + 7) / 8 + (long long)(ffoff[b1] - ffoff[b0]);
        t.out0 = out + header_bytes;
        out = t.out0 + t.stuffed + 2;
        tot[i] = t;
    }
}

__global__ void __launch_bounds__(256) scatter_kernel(const EncImg* __restrict__ imgs, int n, long long nblk,
                                                      const unsigned long long* __restrict__ off,
                                                      const unsigned long long* __restrict__ ffoff, const uint32_t* __restrict__ words,
                                                      const EncTotals* __restrict__ tot, uint8_t* __restrict__ out) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nblk) return;
    const int i = find_image(imgs, n, g);
    const EncImg& I = imgs[i];
    const BitRange r = bit_range(I, i + 1 < n ? &imgs[i + 1] : nullptr, nblk, g, off);
    if (r.b1 > I.bound_bits) return;
    long long b, e;
    owned_bytes(r, &b, &e);
    uint8_t* o = out + tot[i].out0 + b + (long long)(ffoff[g] - ffoff[I.blk0]);
    for (; b < e; b++) {
        const uint8_t v = stream_byte(words + I.word0, b);
        *o++ = v;
        if (v == 0xFF) *o++ = 0;
    }
}

// ---- host -------------------------------------------------------------------------------------------------------------
void huff_codes(const uint8_t* bits, const uint8_t* vals, uint16_t* code, uint8_t* len) {
    int c = 0, k = 0;
    for (int l = 1; l <= 16; l++) {
        for (int j = 0; j < bits[l - 1]; j++, k++) {
            code[vals[k]] = (uint16_t)c++;
            len[vals[k]] = (uint8_t)l;
        }
        c <<= 1;
    }
}

void quant_table(int q, int t, uint8_t* zz_out) {
    const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    for (int i = 0; i < 64; i++) zz_out[i] = (uint8_t)std::min(255, std::max(1, (kBaseQ[t][i] * scale + 50) / 100));
}

void segment(std::vector<uint8_t>* o, uint8_t marker, const std::vector<uint8_t>& body) {
    const size_t L = body.size() + 2;
    o->insert(o->end(), {0xFF, marker, (uint8_t)(L >> 8), (uint8_t)L});
    o->insert(o->end(), body.begin(), body.end());
}

// SOI .. SOS, as libjpeg writes them for cv2's defaults; its length does not depend on the quality or the size
std::vector<uint8_t> jpeg_header(int q, int h, int w) {
    std::vector<uint8_t> o = {0xFF, 0xD8};
    segment(&o, 0xE0, {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
    for (int t = 0; t < 2; t++) {
        std::vector<uint8_t> b(65);
        b[0] = (uint8_t)t;
        quant_table(q, t, b.data() + 1);
        segment(&o, 0xDB, b);
    }
    segment(&o, 0xC0, {8, (uint8_t)(h >> 8), (uint8_t)h, (uint8_t)(w >> 8), (uint8_t)w, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
    for (int t = 0; t < 2; t++) {
        std::vector<uint8_t> dc = {(uint8_t)t};
        dc.insert(dc.end(), kDcBits[t], kDcBits[t] + 16);
        for (int v = 0; v < 12; v++) dc.push_back((uint8_t)v);
        segment(&o, 0xC4, dc);
        std::vector<uint8_t> ac = {(uint8_t)(0x10 | t)};
        ac.insert(ac.end(), kAcBits[t], kAcBits[t] + 16);
        ac.insert(ac.end(), kAcVals[t], kAcVals[t] + 162);
        segment(&o, 0xC4, ac);
    }
    segment(&o, 0xDA, {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
    return o;
}

}  // namespace

struct JpegEncWorkspace {
    PinnedBuffer<uint8_t> host;  // staging: descriptors and tables
    DeviceBuffer<uint8_t> dev_in;
    CompositeStage comp;
    DeviceBuffer<EncTotals> tot;
    PinnedBuffer<EncTotals> tot_host;
    DeviceBuffer<uint8_t> planes;
    DeviceBuffer<int16_t> coef;
    DeviceBuffer<uint32_t> counts;  // bits, then 0xFF bytes, per block
    DeviceBuffer<unsigned long long> off;  // [nblk + 1] bit offsets
    DeviceBuffer<unsigned long long> ffoff;  // [nblk + 1] 0xFF counts before each block
    DeviceBuffer<unsigned long long> tiles;
    DeviceBuffer<uint32_t> words;
    DeviceBuffer<uint8_t> out;
    PinnedBuffer<uint8_t> result;  // the streams of the last call, back to back
    std::vector<int64_t> res_off, res_len;
};

JpegEncWorkspace* jpeg_enc_workspace_create() { return new JpegEncWorkspace(); }

void jpeg_enc_workspace_destroy(JpegEncWorkspace* ws) { delete ws; }

const uint8_t* jpeg_enc_result(const JpegEncWorkspace* ws, int i, int64_t* nbytes) {
    if (!ws || i < 0 || i >= (int)ws->res_off.size()) return nullptr;
    if (nbytes) *nbytes = ws->res_len[i];
    return ws->result + ws->res_off[i];
}

int jpeg_encode(JpegEncWorkspace* ws, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w, int quality,
                const smapb_record* records, const double* scales, int flags, int64_t* nbytes, cudaStream_t st,
                int64_t* launches, std::string* err) {
    ws->res_off.clear();
    ws->res_len.clear();
    if (int rc = composite_args("smapb_encode_jpeg", "smapb_encode_jpeg_ex", n, bgr, img_h, img_w, records, scales, flags, err))
        return rc;
    if (n > 0 && !nbytes) {
        *err = "smapb_encode_jpeg: null argument";
        return -1;
    }
    if (quality < 1 || quality > 100) {
        *err = "smapb_encode_jpeg: quality " + std::to_string(quality) + " outside 1..100";
        return -1;
    }
    if (int rc = composite_frames("smapb_encode_jpeg", "smapb_encode_jpeg_ex", n, bgr, img_h, img_w, flags, err)) return rc;
    if (int rc = refuse_capture("smapb_encode_jpeg", st, err)) return rc;
    if (n == 0) return 0;
    CompositeStage& cs = ws->comp;
    if (int rc = composite_plan(&cs, "smapb_encode_jpeg", n, bgr, img_h, img_w, records, scales, flags, st, err)) return rc;
    std::vector<EncImg> imgs(n);
    long long nblk = 0, plane_total = 0, word_total = 0;
    for (int i = 0; i < n; i++) {
        EncImg& I = imgs[i];
        memset(&I, 0, sizeof(I));
        I.h = cs.imgs[i].h, I.w = cs.imgs[i].w;
        I.mx = (I.w + 15) / 16, I.my = (I.h + 15) / 16, I.bw = (I.w + 7) / 8, I.bh = (I.h + 7) / 8;
        I.blk0 = nblk;
        const long long nb = 6ll * I.mx * I.my;
        nblk += nb;
        I.plane0 = plane_total;
        plane_total += 384ll * I.mx * I.my;
        I.bound_bits = nb * BLOCK_BITS_MAX;
        I.word0 = word_total;
        word_total += (I.bound_bits + 31) / 32 + 1;
    }
    EncTables T;
    memset(&T, 0, sizeof(T));
    for (int t = 0; t < 2; t++) {
        uint8_t q[64];
        quant_table(quality, t, q);
        for (int i = 0; i < 64; i++) T.qdiv[t][kZigzag[i]] = (uint16_t)(8 * q[i]);
        const uint8_t dcv[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
        huff_codes(kDcBits[t], dcv, T.dc_code[t], T.dc_len[t]);
        huff_codes(kAcBits[t], kAcVals[t], T.ac_code[t], T.ac_len[t]);
    }
    const size_t o_tab = align_up(sizeof(EncImg) * n, 256), o_comp = align_up(o_tab + sizeof(EncTables), 256);
    const size_t o_pan = align_up(o_comp + sizeof(Composite) * n, 256);
    const size_t total_in = o_pan + sizeof(PanelImg) * cs.panels.size();
    DECODE_CK(ws->host.grow(total_in));
    memcpy(ws->host, imgs.data(), sizeof(EncImg) * n);
    memcpy(ws->host + o_tab, &T, sizeof(T));
    memcpy(ws->host + o_comp, cs.imgs.data(), sizeof(Composite) * n);
    if (!cs.panels.empty()) memcpy(ws->host + o_pan, cs.panels.data(), sizeof(PanelImg) * n);
    DECODE_CK(ws->dev_in.grow(total_in));
    DECODE_CK(ws->planes.grow((size_t)plane_total));
    DECODE_CK(ws->coef.grow((size_t)nblk * 64));
    DECODE_CK(ws->counts.grow((size_t)nblk));
    DECODE_CK(ws->off.grow((size_t)nblk + 1));
    DECODE_CK(ws->ffoff.grow((size_t)nblk + 1));
    DECODE_CK(ws->words.grow((size_t)word_total));
    DECODE_CK(ws->tot.grow((size_t)n));
    DECODE_CK(ws->tot_host.grow((size_t)n));
    const EncImg* d_img = (const EncImg*)ws->dev_in.get();
    const EncTables* d_tab = (const EncTables*)(ws->dev_in + o_tab);
    const Composite* d_comp = (const Composite*)(ws->dev_in + o_comp);
    DECODE_CK(cudaMemcpyAsync(ws->dev_in, ws->host, total_in, cudaMemcpyHostToDevice, st));
    int max_mcus = 0;
    for (const EncImg& I : imgs) max_mcus = std::max(max_mcus, I.mx * I.my);
    if (int rc = composite_launch(&cs, d_comp, (const PanelImg*)(ws->dev_in + o_pan), n, st, launches, err)) return rc;
    const unsigned fgrid = (unsigned)((nblk + 127) / 128), bgrid = (unsigned)((nblk + 255) / 256);
    colour_kernel<<<dim3((unsigned)((64ll * max_mcus + 255) / 256), n), 256, 0, st>>>(d_img, d_comp, cs.labels, ws->planes);
    fdct_kernel<<<fgrid, 128, 0, st>>>(d_img, n, nblk, d_tab, ws->planes, ws->coef);
    bits_kernel<<<fgrid, 128, 0, st>>>(d_img, n, nblk, d_tab, ws->coef, ws->counts);
    DECODE_CK(cudaGetLastError());
    if (int rc = exclusive_scan(&ws->tiles, ws->counts, nblk, ws->off, st, err)) return rc;
    zero_kernel<<<bgrid, 256, 0, st>>>(d_img, n, nblk, ws->off, ws->words);
    pack_kernel<<<fgrid, 128, 0, st>>>(d_img, n, nblk, d_tab, ws->coef, ws->off, ws->words);
    ff_kernel<<<bgrid, 256, 0, st>>>(d_img, n, nblk, ws->off, ws->words, ws->counts);
    DECODE_CK(cudaGetLastError());
    if (int rc = exclusive_scan(&ws->tiles, ws->counts, nblk, ws->ffoff, st, err)) return rc;
    const std::vector<uint8_t> hdr0 = jpeg_header(quality, 1, 1);
    const long long L = (long long)hdr0.size();
    totals_kernel<<<1, 1, 0, st>>>(d_img, n, nblk, ws->off, ws->ffoff, L, ws->tot);
    DECODE_CK(cudaGetLastError());
    *launches += 13;
    DECODE_CK(cudaMemcpyAsync(ws->tot_host, ws->tot, sizeof(EncTotals) * n, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    long long total_out = 0;
    for (int i = 0; i < n; i++) {
        const EncTotals& t = ws->tot_host[i];
        // the bound the bit buffer was sized by, and the stuffed stream's (every byte stuffed)
        if (t.bits > imgs[i].bound_bits || t.stuffed > 2 * ((imgs[i].bound_bits + 7) / 8)) {
            *err = "smapb_encode_jpeg: frame " + std::to_string(i) + " exceeds the entropy-coded size bound";
            return -1;
        }
        total_out = t.out0 + t.stuffed + 2;
    }
    DECODE_CK(ws->out.grow((size_t)total_out));
    DECODE_CK(ws->result.grow((size_t)total_out));
    scatter_kernel<<<bgrid, 256, 0, st>>>(d_img, n, nblk, ws->off, ws->ffoff, ws->words, ws->tot, ws->out);
    DECODE_CK(cudaGetLastError());
    ++*launches;
    DECODE_CK(cudaMemcpyAsync(ws->result, ws->out, (size_t)total_out, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    for (int i = 0; i < n; i++) {
        const EncTotals& t = ws->tot_host[i];
        const std::vector<uint8_t> hdr = jpeg_header(quality, imgs[i].h, imgs[i].w);
        memcpy(ws->result + t.out0 - L, hdr.data(), L);
        ws->result[t.out0 + t.stuffed] = 0xFF;
        ws->result[t.out0 + t.stuffed + 1] = 0xD9;
        ws->res_off.push_back(t.out0 - L);
        ws->res_len.push_back(L + t.stuffed + 2);
        nbytes[i] = L + t.stuffed + 2;
    }
    return 0;
}

}  // namespace smapb
