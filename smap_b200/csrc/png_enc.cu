// PNG encoding on the GPU, byte-identical to cv2.imencode(".png", bgr) (libpng with zlib at level 1, memLevel 8 and
// strategy Z_RLE; rules in include/smap_b200.h, smapb_encode_png), restated stage by stage on the CPU by
// oracle/png_encode_numpy.py.
//
// Z_RLE only ever looks one byte back, so zlib's token stream needs no dictionary search: inside each maximal run of
// equal bytes the first byte is a literal, then come 258-long matches at distance 1, then one shorter match (3..257) or
// up to 2 literals.  Every phase is one launch for the whole batch (frames of any sizes):
//   overlay   (records only) the composite stage's label planes (overlay.cuh, view3d.cu);
//   filter    one thread per pixel: the composite pixel as RGB, minus the pixel to its left (Sub), and the row's filter
//             byte (None when W = 1);
//   runs      one thread per byte: does a run of equal bytes start here (every image's first byte does)?  An exclusive
//             scan (scan.cuh, three launches) numbers the runs, and `runpos` scatters each run's first byte;
//   parse     one thread per byte: from its run's start and end, is a symbol (literal or match) emitted here?  A second
//             scan numbers the symbols, and `compact` stores them and the first byte of every 16383-symbol block;
//   histogram one CTA per block counts its literal/length codes in shared memory;
//   trees     one thread per block runs zlib's trees.c: code lengths, codes, the stored / fixed / dynamic choice and the
//             block's size in bits;
//   adler     the Adler-32 of each image, from per-CTA sums combined with atomics;
//   walk      one thread per image walks its blocks in order (a stored block's padding depends on the bit position),
//             writes the zlib header and the Adler-32, and thread 0 lays out the files;
//   emit      one CTA per block: its header by one thread, its symbols from a CTA-wide scan of their lengths, stored
//             bytes word by word; words shared with a neighbour are merged with atomicOr, so the stream does not depend
//             on the order;
//   frame     (after one D2H of the sizes) one CTA per IDAT chunk copies its bytes into the file and computes its CRC-32.
// One D2H brings the files back; the host writes the signature, IHDR and IEND.
#include <string.h>

#include <algorithm>
#include <vector>

#include "checksum.cuh"
#include "decode_host.h"
#include "overlay.cuh"
#include "png_enc.h"
#include "scan.cuh"

namespace smapb {

namespace {

constexpr int BLOCK_SYMS = 16383;  // zlib flushes a block every lit_bufsize - 1 symbols (memLevel 8)
constexpr int IDAT_BYTES = 8192;  // libpng cuts the zlib stream into chunks of this size
constexpr int L_CODES = 286, D_CODES = 30, BL_CODES = 19, HEAP_SIZE = 2 * L_CODES + 1;
constexpr int MAX_MATCH = 258, MIN_LOOKAHEAD = 262;
constexpr int EMIT_THREADS = SCAN_THREADS;  // the emit CTA scans with block_exclusive
constexpr int FRAME_THREADS = 256;
constexpr uint16_t NO_SYMBOL = 0xFFFF;

__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t kLenBase[29] = {0,  1,  2,  3,  4,  5,  6,   7,   8,   10,  12,  14,  16,  20, 24,
                                     28, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 255};
__constant__ uint8_t kDistExtra[D_CODES] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kBlExtra[BL_CODES] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ uint8_t kBlOrder[BL_CODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct PngImg {
    int h, w;  // the composite's size
    long long n;  // filtered stream bytes: h (1 + 3 w)
    long long raw0;  // its first byte in the batch's stream
    long long blk0;  // its first block record
    int blk_cap;  // n / 16383 + 1 (every symbol covers at least one byte)
    int wsize;  // zlib's window: 1 << windowBits
    int cmf, flg;  // the zlib header
    long long z0, zcap;  // its zlib stream's first byte in the stream buffer, and the bytes reserved there
};

struct ImgOut {
    long long zlen;  // zlib stream bytes; -1: more than zcap (refused)
    long long file0;  // the file's first byte in the output
    long long chunk0;  // its first IDAT chunk in the batch
    long long chunks;  // IDAT chunks of the whole batch (image 0 only)
};

struct Blk {
    long long first, flush;  // (compact) the first symbol's byte, and the last one's in a block that is not the last
    long long pos0;  // the block's first byte
    long long sym0, bit0;  // first symbol (batch), first bit in the image's zlib stream
    long long bits;  // the block's size in bits (stored: without the padding to the byte boundary)
    int nsym, stored_len, type, last;  // type: 0 stored, 1 fixed, 2 dynamic, -1 past the image's blocks
    int lcodes, dcodes, blcodes;
    uint16_t lcode[L_CODES], dcode[D_CODES], blcode[BL_CODES];
    uint8_t llen[L_CODES], dlen[D_CODES], bllen[BL_CODES];
};

template <typename Key>
__device__ __forceinline__ int find_image(const PngImg* im, int n, long long g, Key key) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (key(im[mid]) <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ int image_of_byte(const PngImg* im, int n, long long g) {
    return find_image(im, n, g, [](const PngImg& I) { return I.raw0; });
}

// ---- filter ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) filter_kernel(const PngImg* __restrict__ imgs, const Composite* __restrict__ comps,
                                                     const int* __restrict__ labels, uint8_t* __restrict__ raw) {
    const PngImg& I = imgs[blockIdx.y];
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (long long)I.w * I.h) return;
    const int x = (int)(k % I.w), y = (int)(k / I.w);
    int b, g, r, pb = 0, pg = 0, pr = 0;
    load_pixel(comps[blockIdx.y], labels, x, y, &b, &g, &r);
    if (I.w > 1 && x > 0) load_pixel(comps[blockIdx.y], labels, x - 1, y, &pb, &pg, &pr);
    uint8_t* row = raw + I.raw0 + (long long)y * (1 + 3ll * I.w);
    if (x == 0) row[0] = I.w > 1 ? 1 : 0;
    row[1 + 3 * x] = (uint8_t)(r - pr), row[2 + 3 * x] = (uint8_t)(g - pg), row[3 + 3 * x] = (uint8_t)(b - pb);
}

// ---- runs and the parse ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool run_start(const PngImg& I, const uint8_t* raw, long long g) {
    return g == I.raw0 || raw[g] != raw[g - 1];
}

__global__ void __launch_bounds__(256) runs_kernel(const PngImg* __restrict__ imgs, int n, long long total,
                                                   const uint8_t* __restrict__ raw, uint32_t* __restrict__ flag) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    flag[g] = run_start(imgs[image_of_byte(imgs, n, g)], raw, g);
}

__global__ void __launch_bounds__(256) runpos_kernel(const PngImg* __restrict__ imgs, int n, long long total,
                                                     const uint8_t* __restrict__ raw, const unsigned long long* __restrict__ runx,
                                                     long long* __restrict__ runpos) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    if (run_start(imgs[image_of_byte(imgs, n, g)], raw, g)) runpos[runx[g]] = g;
    if (g == total - 1) runpos[runx[total]] = total;  // the end of the last run
}

// The symbol starting at byte g, or NO_SYMBOL: a run [a, b) of equal bytes is a literal at a, then matches of 258 at
// a + 1 + 258 j while at least 258 bytes are left, then a match of the rest m when m >= 3, else m literals.
__device__ __forceinline__ uint16_t symbol_at(const uint8_t* raw, long long g, long long a, long long b) {
    if (g == a) return raw[g];
    const long long k = g - a - 1, r = b - a - 1, q = r / MAX_MATCH, m = r % MAX_MATCH;
    if (k < q * MAX_MATCH) return k % MAX_MATCH == 0 ? (uint16_t)(256 + MAX_MATCH - 3) : NO_SYMBOL;
    if (m >= 3) return k == q * MAX_MATCH ? (uint16_t)(256 + m - 3) : NO_SYMBOL;
    return raw[g];
}

__global__ void __launch_bounds__(256) parse_kernel(const PngImg* __restrict__ imgs, int n, long long total,
                                                    const uint8_t* __restrict__ raw, const unsigned long long* __restrict__ runx,
                                                    const long long* __restrict__ runpos, uint16_t* __restrict__ tok,
                                                    uint32_t* __restrict__ count) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const bool start = run_start(imgs[image_of_byte(imgs, n, g)], raw, g);
    const unsigned long long r = runx[g] + start - 1;
    const uint16_t s = symbol_at(raw, g, runpos[r], runpos[r + 1]);
    tok[g] = s;
    count[g] = s != NO_SYMBOL;
}

__global__ void __launch_bounds__(256) compact_kernel(const PngImg* __restrict__ imgs, int n, long long total,
                                                      const uint16_t* __restrict__ tok, const unsigned long long* __restrict__ symx,
                                                      uint16_t* __restrict__ sym, Blk* __restrict__ blks) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total || tok[g] == NO_SYMBOL) return;
    const PngImg& I = imgs[image_of_byte(imgs, n, g)];
    const unsigned long long s = symx[g], local = s - symx[I.raw0];
    sym[s] = tok[g];
    Blk& B = blks[I.blk0 + (long long)(local / BLOCK_SYMS)];
    if (local % BLOCK_SYMS == 0) B.first = g - I.raw0;
    if (local % BLOCK_SYMS == BLOCK_SYMS - 1) B.flush = g - I.raw0;
}

// ---- blocks -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int image_of_block(const PngImg* im, int n, long long b) {
    return find_image(im, n, b, [](const PngImg& I) { return I.blk0; });
}

// the image's symbol count, from the symbol scan
__device__ __forceinline__ long long image_symbols(const PngImg& I, const unsigned long long* symx) {
    return (long long)(symx[I.raw0 + I.n] - symx[I.raw0]);
}

// the length code (257..285) of match length - 3 = l
__device__ __forceinline__ int length_code(int l) {
    int c = 284;
    if (l == 255) return 285;
    while (kLenBase[c - 257] > l) c--;
    return c;
}

__global__ void __launch_bounds__(256) histogram_kernel(const PngImg* __restrict__ imgs, int n, const unsigned long long* __restrict__ symx,
                                                        const uint16_t* __restrict__ sym, uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[L_CODES];
    const long long gb = blockIdx.x;
    const PngImg& I = imgs[image_of_block(imgs, n, gb)];
    for (int i = threadIdx.x; i < L_CODES; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const long long ns = image_symbols(I, symx), s0 = (gb - I.blk0) * BLOCK_SYMS, s1 = min(ns, s0 + BLOCK_SYMS);
    const unsigned long long base = symx[I.raw0];
    for (long long s = s0 + threadIdx.x; s < s1; s += blockDim.x) {
        const int v = sym[base + s];
        atomicAdd(&h[v < 256 ? v : length_code(v - 256)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < L_CODES; i += blockDim.x) hist[gb * L_CODES + i] = h[i];
}

// zlib's build_tree + gen_bitlen + gen_codes for one tree: lengths and bit-reversed codes of symbols 0..elems-1, its
// max_code, and what it adds to opt_len and static_len (stree: the static tree's lengths, or NULL).
struct Tree {
    int max_code;
    long long opt, stat;
};

__device__ __noinline__ Tree build_tree(const uint32_t* freq, int elems, const uint8_t* stree, const uint8_t* extra, int base,
                                        int max_length, uint8_t* len_out, uint16_t* code_out) {
    uint32_t f[HEAP_SIZE];
    uint16_t dad[HEAP_SIZE], heap[HEAP_SIZE + 1];
    uint8_t depth[HEAP_SIZE], len[HEAP_SIZE];
    Tree T{-1, 0, 0};
    int heap_len = 0, heap_max = HEAP_SIZE;
    for (int i = 0; i < elems; i++) {
        f[i] = freq[i];
        len[i] = 0;
        depth[i] = 0;
        if (f[i]) heap[++heap_len] = (uint16_t)(T.max_code = i);
    }
    while (heap_len < 2) {  // at least two codes
        const int node = T.max_code < 2 ? ++T.max_code : 0;
        heap[++heap_len] = (uint16_t)node;
        f[node] = 1;
        depth[node] = 0;
        T.opt--;
        if (stree) T.stat -= stree[node];
    }
    auto smaller = [&](int a, int b) { return f[a] < f[b] || (f[a] == f[b] && depth[a] <= depth[b]); };
    auto down = [&](int k) {
        const int v = heap[k];
        int j = k << 1;
        while (j <= heap_len) {
            if (j < heap_len && smaller(heap[j + 1], heap[j])) j++;
            if (smaller(v, heap[j])) break;
            heap[k] = heap[j];
            k = j;
            j <<= 1;
        }
        heap[k] = (uint16_t)v;
    };
    for (int k = heap_len / 2; k >= 1; k--) down(k);
    int node = elems;
    do {
        const int a = heap[1];
        heap[1] = heap[heap_len--];
        down(1);
        const int b = heap[1];
        heap[--heap_max] = (uint16_t)a;
        heap[--heap_max] = (uint16_t)b;
        f[node] = f[a] + f[b];
        depth[node] = (uint8_t)(max(depth[a], depth[b]) + 1);
        dad[a] = dad[b] = (uint16_t)node;
        heap[1] = (uint16_t)node++;
        down(1);
    } while (heap_len >= 2);
    heap[--heap_max] = heap[1];
    // gen_bitlen
    int bl_count[16] = {0};
    len[heap[heap_max]] = 0;
    int overflow = 0, h;
    for (h = heap_max + 1; h < HEAP_SIZE; h++) {
        const int m = heap[h];
        int bits = len[dad[m]] + 1;
        if (bits > max_length) bits = max_length, overflow++;
        len[m] = (uint8_t)bits;
        if (m > T.max_code) continue;
        bl_count[bits]++;
        const int xb = m >= base ? extra[m - base] : 0;
        T.opt += (long long)f[m] * (bits + xb);
        if (stree) T.stat += (long long)f[m] * (stree[m] + xb);
    }
    if (overflow) {
        do {
            int bits = max_length - 1;
            while (bl_count[bits] == 0) bits--;
            bl_count[bits]--;
            bl_count[bits + 1] += 2;
            bl_count[max_length]--;
            overflow -= 2;
        } while (overflow > 0);
        for (int bits = max_length; bits != 0; bits--) {
            int c = bl_count[bits];
            while (c != 0) {
                const int m = heap[--h];
                if (m > T.max_code) continue;
                if (len[m] != bits) {
                    T.opt += ((long long)bits - len[m]) * f[m];
                    len[m] = (uint8_t)bits;
                }
                c--;
            }
        }
    }
    // gen_codes
    int next[16], code = 0;
    for (int bits = 1; bits <= 15; bits++) next[bits] = code = (code + bl_count[bits - 1]) << 1;
    for (int i = 0; i < elems; i++) {
        len_out[i] = i <= T.max_code ? len[i] : 0;
        code_out[i] = len_out[i] ? (uint16_t)(__brev(next[len_out[i]]++) >> (32 - len_out[i])) : 0;
    }
    return T;
}

// scan_tree / send_tree: calls put(symbol, extra value, extra bits) for the code-length sequence of lens[0..max_code]
template <typename Put>
__device__ __forceinline__ void tree_runs(const uint8_t* lens, int max_code, Put put) {
    int prevlen = -1, nextlen = lens[0], count = 0;
    int max_count = nextlen == 0 ? 138 : 7, min_count = nextlen == 0 ? 3 : 4;
    for (int i = 0; i <= max_code; i++) {
        const int curlen = nextlen;
        nextlen = i + 1 <= max_code ? lens[i + 1] : 0xFFFF;  // zlib's guard
        if (++count < max_count && curlen == nextlen) continue;
        if (count < min_count) {
            for (; count; count--) put(curlen, 0, 0);
        } else if (curlen != 0) {
            if (curlen != prevlen) put(curlen, 0, 0), count--;
            put(16, count - 3, 2);
        } else if (count <= 10) {
            put(17, count - 3, 3);
        } else {
            put(18, count - 11, 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

// Bytes slid out of zlib's window when its loop reaches position p of n (oracle/png_encode_numpy.py, window_offset).
__device__ __forceinline__ long long window_offset(long long p, long long n, long long wsize) {
    const long long ka = max(0ll, (n - 1) / wsize - 1);
    long long cnt = min(ka, max(0ll, (p + MAX_MATCH) / wsize - 1));
    if (cnt == ka && p >= max(n - MAX_MATCH, (ka + 2) * wsize - MIN_LOOKAHEAD)) cnt++;
    return cnt * wsize;
}

__device__ __forceinline__ int static_llen(int i) { return i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8; }

// the fixed Huffman codes (RFC 1951 3.2.6)
__device__ __forceinline__ void fixed_codes(Blk& B) {
    int next[4] = {0x30, 0x190, 0, 0xC0};  // first codes of 0..143 (8 bits), 144..255 (9), 256..279 (7), 280.. (8)
    for (int i = 0; i < L_CODES; i++) {
        const int k = i < 144 ? 0 : i < 256 ? 1 : i < 280 ? 2 : 3, l = static_llen(i);
        B.llen[i] = (uint8_t)l;
        B.lcode[i] = (uint16_t)(__brev(next[k]++) >> (32 - l));
    }
    for (int i = 0; i < D_CODES; i++) B.dlen[i] = 5, B.dcode[i] = (uint16_t)(__brev(i) >> 27);
}

__global__ void __launch_bounds__(64) trees_kernel(const PngImg* __restrict__ imgs, int n, long long nblk,
                                                   const unsigned long long* __restrict__ symx, const uint32_t* __restrict__ hist,
                                                   Blk* __restrict__ blks) {
    const long long gb = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gb >= nblk) return;
    const PngImg& I = imgs[image_of_block(imgs, n, gb)];
    Blk& B = blks[gb];
    const long long ns = image_symbols(I, symx), b = gb - I.blk0, nb = ns / BLOCK_SYMS + 1;
    if (b >= nb) {
        B.type = -1;
        return;
    }
    const long long s0 = b * BLOCK_SYMS;
    B.last = b == nb - 1;
    B.nsym = (int)min((long long)BLOCK_SYMS, ns - s0);
    B.sym0 = (long long)symx[I.raw0] + s0;
    const long long pos0 = B.nsym ? B.first : I.n;
    const long long pos1 = !B.last && s0 + BLOCK_SYMS < ns ? blks[gb + 1].first : I.n;
    const long long flush = B.last ? I.n : B.flush;
    B.pos0 = pos0;
    B.stored_len = (int)(pos1 - pos0);
    uint32_t lf[L_CODES], df[D_CODES] = {0}, bf[BL_CODES] = {0};
    for (int i = 0; i < L_CODES; i++) lf[i] = hist[gb * L_CODES + i];
    lf[256] = 1;  // END_BLOCK
    for (int i = 257; i < L_CODES; i++) df[0] += lf[i];
    uint8_t sl[L_CODES], sd[D_CODES];
    for (int i = 0; i < L_CODES; i++) sl[i] = (uint8_t)static_llen(i);
    for (int i = 0; i < D_CODES; i++) sd[i] = 5;
    const Tree lt = build_tree(lf, L_CODES, sl, kLenExtra, 257, 15, B.llen, B.lcode);
    const Tree dt = build_tree(df, D_CODES, sd, kDistExtra, 0, 15, B.dlen, B.dcode);
    auto count = [&](int s, int, int) { bf[s]++; };
    tree_runs(B.llen, lt.max_code, count);
    tree_runs(B.dlen, dt.max_code, count);
    const Tree bt = build_tree(bf, BL_CODES, nullptr, kBlExtra, 0, 7, B.bllen, B.blcode);
    int max_blindex = BL_CODES - 1;
    for (; max_blindex >= 3; max_blindex--)
        if (B.bllen[kBlOrder[max_blindex]] != 0) break;
    const long long opt = lt.opt + dt.opt + bt.opt + 3 * (max_blindex + 1) + 14, stat = lt.stat + dt.stat;
    long long opt_lenb = (opt + 3 + 7) >> 3;
    const long long static_lenb = (stat + 3 + 7) >> 3;
    if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
    const bool in_window = pos0 - window_offset(flush, I.n, I.wsize) >= 0;
    if (B.stored_len + 4 <= opt_lenb && in_window) {
        B.type = 0;
        B.bits = 3 + 32 + 8ll * B.stored_len;
    } else if (static_lenb == opt_lenb) {
        B.type = 1;
        B.bits = stat + 3;
        fixed_codes(B);
    } else {
        B.type = 2;
        B.bits = opt + 3;
        B.lcodes = lt.max_code + 1, B.dcodes = dt.max_code + 1, B.blcodes = max_blindex + 1;
    }
}

// ---- Adler-32, the block walk and the file layout ------------------------------------------------------------------
constexpr int ADLER_TILE = 4096;

__global__ void __launch_bounds__(256) adler_kernel(const PngImg* __restrict__ imgs, const uint8_t* __restrict__ raw,
                                                    unsigned long long* __restrict__ sums) {
    __shared__ unsigned long long red[2][8];
    const PngImg& I = imgs[blockIdx.y];
    const long long t0 = (long long)blockIdx.x * ADLER_TILE;
    if (t0 >= I.n) return;
    unsigned long long s1 = 0, s2 = 0;  // sum of bytes, sum of (n - i) * byte
    for (long long i = t0 + threadIdx.x; i < min(I.n, t0 + ADLER_TILE); i += blockDim.x) {
        const unsigned v = raw[I.raw0 + i];
        s1 += v;
        s2 += (unsigned long long)(I.n - i) * v;
    }
    for (int o = 16; o; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o), s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = s1, red[1][threadIdx.x >> 5] = s2;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long a = 0, b = 0;
        for (int w = 0; w < 8; w++) a += red[0][w], b += red[1][w] % ADLER_MOD;
        atomicAdd(&sums[2 * blockIdx.y], a % ADLER_MOD);
        atomicAdd(&sums[2 * blockIdx.y + 1], b % ADLER_MOD);
    }
}

__device__ __forceinline__ long long file_bytes(long long zlen) { return 8 + 25 + 12 * ((zlen + IDAT_BYTES - 1) / IDAT_BYTES) + zlen + 12; }

__global__ void __launch_bounds__(256) walk_kernel(const PngImg* __restrict__ imgs, int n, Blk* __restrict__ blks,
                                                   const unsigned long long* __restrict__ sums, uint8_t* __restrict__ zs,
                                                   ImgOut* __restrict__ out) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const PngImg& I = imgs[i];
        long long bit = 16;
        for (long long b = I.blk0; b < I.blk0 + I.blk_cap && blks[b].type >= 0; b++) {
            Blk& B = blks[b];
            B.bit0 = bit;
            bit = B.type == 0 ? ((bit + 3 + 7) & ~7ll) + 32 + 8ll * B.stored_len : bit + B.bits;
        }
        const long long zbytes = (bit + 7) >> 3;
        uint8_t* z = zs + I.z0;
        if (zbytes + 4 > I.zcap) {
            out[i].zlen = -1;
            continue;
        }
        out[i].zlen = zbytes + 4;
        z[0] = (uint8_t)I.cmf, z[1] = (uint8_t)I.flg;
        const uint32_t a = (uint32_t)((1 + sums[2 * i]) % ADLER_MOD), s = (uint32_t)((I.n + sums[2 * i + 1]) % ADLER_MOD);
        const uint32_t adler = s << 16 | a;
        for (int k = 0; k < 4; k++) z[zbytes + k] = (uint8_t)(adler >> (24 - 8 * k));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long file = 0, chunk = 0;
        for (int i = 0; i < n; i++) {
            const long long zl = max(out[i].zlen, 0ll);
            out[i].file0 = file, out[i].chunk0 = chunk;
            file += file_bytes(zl);
            chunk += (zl + IDAT_BYTES - 1) / IDAT_BYTES;
        }
        out[0].chunks = chunk;
    }
}

// ---- emit ---------------------------------------------------------------------------------------------------------
// LSB-first bit writer over the image's words: the first and the last word it touches are merged with atomicOr, the words
// in between are its own
struct BitWriter {
    uint32_t* W;
    long long wi;
    int nacc;
    unsigned long long acc;
    bool first;
    __device__ BitWriter(uint32_t* words, long long bit) : W(words), wi(bit >> 5), nacc((int)(bit & 31)), acc(0), first(true) {}
    __device__ __forceinline__ void put(uint32_t v, int len) {
        acc |= (unsigned long long)v << nacc;
        nacc += len;
        if (nacc >= 32) {
            if (first) atomicOr(&W[wi], (uint32_t)acc);
            else W[wi] = (uint32_t)acc;
            first = false;
            acc >>= 32;
            nacc -= 32;
            wi++;
        }
    }
    __device__ __forceinline__ void flush() {
        if (nacc > 0) atomicOr(&W[wi], (uint32_t)acc);
    }
};

// a symbol's code, extra bits and distance code: (bits, length); at most 15 + 5 + 5 bits, as the distance tree is either
// the fixed one or two forced codes of length 1
__device__ __forceinline__ void symbol_bits(const Blk& B, int v, uint32_t* bits, int* len) {
    if (v < 256) {
        *bits = B.lcode[v], *len = B.llen[v];
        return;
    }
    const int l = v - 256, c = length_code(l), xb = kLenExtra[c - 257], ll = B.llen[c];
    *bits = B.lcode[c] | (uint32_t)(l - kLenBase[c - 257]) << ll | (uint32_t)B.dcode[0] << (ll + xb);
    *len = ll + xb + B.dlen[0];
}

__global__ void __launch_bounds__(EMIT_THREADS) emit_kernel(const PngImg* __restrict__ imgs, int n, const Blk* __restrict__ blks,
                                                            const uint16_t* __restrict__ sym, const uint8_t* __restrict__ raw,
                                                            const ImgOut* __restrict__ out, uint8_t* __restrict__ zs) {
    __shared__ long long s_data;  // the first bit of the block's symbols
    const long long gb = blockIdx.x;
    const int im = image_of_block(imgs, n, gb);
    const PngImg& I = imgs[im];
    const Blk& B = blks[gb];
    if (B.type < 0 || out[im].zlen < 0) return;
    uint32_t* W = reinterpret_cast<uint32_t*>(zs + I.z0);  // z0 is word-aligned
    if (threadIdx.x == 0) {
        BitWriter w(W, B.bit0);
        w.put(B.type << 1 | B.last, 3);
        if (B.type == 2) {
            w.put(B.lcodes - 257, 5);
            w.put(B.dcodes - 1, 5);
            w.put(B.blcodes - 4, 4);
            for (int i = 0; i < B.blcodes; i++) w.put(B.bllen[kBlOrder[i]], 3);
            auto send = [&](int s, int xv, int xb) {
                w.put(B.blcode[s], B.bllen[s]);
                if (xb) w.put(xv, xb);
            };
            tree_runs(B.llen, B.lcodes - 1, send);
            tree_runs(B.dlen, B.dcodes - 1, send);
        }
        w.flush();
        s_data = 32 * w.wi + w.nacc;
    }
    __syncthreads();
    if (B.type == 0) {  // LEN, NLEN and the bytes, from the byte after the 3 header bits
        const long long p = (B.bit0 + 3 + 7) >> 3, end = p + 4 + B.stored_len;
        const uint8_t* src = raw + I.raw0 + B.pos0;
        for (long long wi = (p >> 2) + threadIdx.x; 4 * wi < end; wi += blockDim.x) {
            uint32_t v = 0;
            bool whole = true;
            for (int k = 0; k < 4; k++) {
                const long long q = 4 * wi + k;
                uint32_t byte = 0;
                if (q < p || q >= end) whole = false;
                else if (q < p + 2) byte = (uint32_t)(B.stored_len >> (8 * (q - p))) & 255;
                else if (q < p + 4) byte = (uint32_t)(~B.stored_len >> (8 * (q - p - 2))) & 255;
                else byte = src[q - p - 4];
                v |= byte << (8 * k);
            }
            if (whole) W[wi] = v;
            else atomicOr(&W[wi], v);
        }
        return;
    }
    // each thread a run of consecutive symbols, placed by a CTA-wide scan of their lengths
    const int per = (B.nsym + EMIT_THREADS - 1) / EMIT_THREADS;
    const int k0 = min(B.nsym, (int)threadIdx.x * per), k1 = min(B.nsym, k0 + per);
    const uint16_t* S = sym + B.sym0;
    unsigned long long mine = 0;
    for (int k = k0; k < k1; k++) {
        uint32_t v;
        int len;
        symbol_bits(B, S[k], &v, &len);
        mine += len;
    }
    unsigned long long total;
    const unsigned long long before = block_exclusive(mine, &total);
    if (k1 > k0) {
        BitWriter w(W, s_data + (long long)before);
        for (int k = k0; k < k1; k++) {
            uint32_t v;
            int len;
            symbol_bits(B, S[k], &v, &len);
            w.put(v, len);
        }
        w.flush();
    }
    if (threadIdx.x == 0) {
        BitWriter w(W, s_data + (long long)total);
        w.put(B.lcode[256], B.llen[256]);
        w.flush();
    }
}

// ---- frame ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

__global__ void __launch_bounds__(FRAME_THREADS) frame_kernel(const PngImg* __restrict__ imgs, int n, const ImgOut* __restrict__ out,
                                                              const uint8_t* __restrict__ zs, uint8_t* __restrict__ file) {
    __shared__ uint32_t T[256], x2n[32], red[FRAME_THREADS / 32];
    crc_tables(T, x2n);
    const long long c = blockIdx.x;
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (out[mid].chunk0 <= c) lo = mid;
        else hi = mid - 1;
    }
    const PngImg& I = imgs[lo];
    const ImgOut& O = out[lo];
    const long long k = c - O.chunk0, d0 = k * IDAT_BYTES, len = min((long long)IDAT_BYTES, O.zlen - d0);
    uint8_t* f = file + O.file0 + 33 + k * (IDAT_BYTES + 12);
    const uint8_t* z = zs + I.z0 + d0;
    for (long long j = threadIdx.x; j < len; j += blockDim.x) f[8 + j] = z[j];
    const uint8_t kIdat[4] = {'I', 'D', 'A', 'T'};
    uint32_t r = crc_slice(T, x2n, 4 + len, [&](uint64_t j) { return j < 4 ? kIdat[j] : z[j - 4]; });
    for (int o = 16; o; o >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < FRAME_THREADS / 32; w++) t ^= red[w];
        put_be32(f, (uint32_t)len);
        for (int i = 0; i < 4; i++) f[4 + i] = kIdat[i];
        put_be32(f + 8 + len, crc_finish(x2n, 4 + len, t));
    }
}

// ---- host -------------------------------------------------------------------------------------------------------------
// zlib's windowBits as libpng sets it for n bytes of scanlines, and the header after libpng's CINFO rewrite
void zlib_header(long long n, int* wsize, int* cmf, int* flg) {
    int wbits = 15;
    if (n <= 16384) {
        for (long long half = 16384; n + MIN_LOOKAHEAD <= half; half >>= 1) wbits--;
    }
    *wsize = 1 << wbits;
    int c = 8 | (wbits - 8) << 4;
    if (n <= 16384) {
        int cinfo = c >> 4;
        long long half = 1ll << (cinfo + 7);
        if (n <= half) {
            do {
                half >>= 1;
                cinfo--;
            } while (cinfo > 0 && n <= half);
            c = (c & 15) | cinfo << 4;
        }
    }
    *cmf = c;
    *flg = 31 - (c * 256) % 31;
}

void put_be32_host(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

// the 12 bytes of chunk `type` with `len` bytes of data at p + 8 (already there)
void host_chunk(uint8_t* p, const char* type, uint32_t len) {
    put_be32_host(p, len);
    memcpy(p + 4, type, 4);
    put_be32_host(p + 8 + len, crc32_host(p + 4, 4 + (int64_t)len));
}

}  // namespace

struct PngEncWorkspace {
    PinnedBuffer<uint8_t> host;  // staging: descriptors
    DeviceBuffer<uint8_t> dev_in;
    CompositeStage comp;
    DeviceBuffer<uint8_t> raw;  // the filtered streams
    DeviceBuffer<uint32_t> counts;  // run starts, then symbols, per byte
    DeviceBuffer<unsigned long long> x;  // [total + 1] runs, then symbols, before each byte
    DeviceBuffer<unsigned long long> tiles;
    DeviceBuffer<long long> runpos;  // [runs + 1] first byte of each run
    DeviceBuffer<uint16_t> tok, sym;
    DeviceBuffer<uint32_t> hist;  // [blocks][286]
    DeviceBuffer<Blk> blks;
    DeviceBuffer<unsigned long long> sums;  // [n][2] Adler-32 sums
    DeviceBuffer<ImgOut> out;
    PinnedBuffer<ImgOut> out_host;
    DeviceBuffer<uint8_t> zs;  // the zlib streams
    DeviceBuffer<uint8_t> file;
    PinnedBuffer<uint8_t> result;  // the files of the last call, back to back
    std::vector<int64_t> res_off, res_len;
};

PngEncWorkspace* png_enc_workspace_create() { return new PngEncWorkspace(); }

void png_enc_workspace_destroy(PngEncWorkspace* ws) { delete ws; }

const uint8_t* png_enc_result(const PngEncWorkspace* ws, int i, int64_t* nbytes) {
    if (!ws || i < 0 || i >= (int)ws->res_off.size()) return nullptr;
    if (nbytes) *nbytes = ws->res_len[i];
    return ws->result + ws->res_off[i];
}

int png_encode(PngEncWorkspace* ws, int n, const uint8_t* const* bgr, const int* img_h, const int* img_w,
               const smapb_record* records, const double* scales, int flags, int64_t* nbytes, cudaStream_t st,
               int64_t* launches, std::string* err) {
    const char* kCall = "smapb_encode_png";
    if (int rc = composite_args(kCall, kCall, n, bgr, img_h, img_w, records, scales, flags, err)) return rc;
    if (n > 0 && !nbytes) {
        *err = std::string(kCall) + ": null argument";
        return -1;
    }
    if (int rc = composite_frames(kCall, kCall, n, bgr, img_h, img_w, flags, err)) return rc;
    if (int rc = refuse_capture(kCall, st, err)) return rc;
    CompositeStage& cs = ws->comp;
    if (n > 0)
        if (int rc = composite_plan(&cs, kCall, n, bgr, img_h, img_w, records, scales, flags, st, err)) return rc;
    ws->res_off.clear();
    ws->res_len.clear();
    if (n == 0) return 0;
    std::vector<PngImg> imgs(n);
    long long total = 0, nblk = 0, ztotal = 0;
    int max_pix = 0;
    long long max_n = 0;
    for (int i = 0; i < n; i++) {
        PngImg& I = imgs[i];
        memset(&I, 0, sizeof(I));
        I.h = cs.imgs[i].h, I.w = cs.imgs[i].w;
        I.n = (long long)I.h * (1 + 3ll * I.w);
        I.raw0 = total;
        total += I.n;
        I.blk0 = nblk;
        I.blk_cap = (int)(I.n / BLOCK_SYMS + 1);
        nblk += I.blk_cap;
        zlib_header(I.n, &I.wsize, &I.cmf, &I.flg);
        // a block costs at most its fixed-code size (9 bits per byte) or, stored, its bytes: + 10 bits of type and END,
        // padding, LEN / NLEN
        I.zcap = align_up((size_t)(6 + I.n * 9 / 8 + 8ll * I.blk_cap + 64), 16);
        I.z0 = ztotal;
        ztotal += I.zcap;
        max_pix = std::max(max_pix, I.h * I.w);
        max_n = std::max(max_n, I.n);
    }
    const size_t o_comp = align_up(sizeof(PngImg) * n, 256), o_pan = align_up(o_comp + sizeof(Composite) * n, 256);
    const size_t total_in = o_pan + sizeof(PanelImg) * cs.panels.size();
    DECODE_CK(ws->host.grow(total_in));
    memcpy(ws->host, imgs.data(), sizeof(PngImg) * n);
    memcpy(ws->host + o_comp, cs.imgs.data(), sizeof(Composite) * n);
    if (!cs.panels.empty()) memcpy(ws->host + o_pan, cs.panels.data(), sizeof(PanelImg) * n);
    DECODE_CK(ws->dev_in.grow(total_in));
    DECODE_CK(ws->raw.grow((size_t)total));
    DECODE_CK(ws->counts.grow((size_t)total));
    DECODE_CK(ws->x.grow((size_t)total + 1));
    DECODE_CK(ws->runpos.grow((size_t)total + 1));
    DECODE_CK(ws->tok.grow((size_t)total));
    DECODE_CK(ws->sym.grow((size_t)total));
    DECODE_CK(ws->hist.grow((size_t)nblk * L_CODES));
    DECODE_CK(ws->blks.grow((size_t)nblk));
    DECODE_CK(ws->sums.grow((size_t)2 * n));
    DECODE_CK(ws->out.grow((size_t)n));
    DECODE_CK(ws->out_host.grow((size_t)n));
    DECODE_CK(ws->zs.grow((size_t)ztotal));
    const PngImg* d_img = (const PngImg*)ws->dev_in.get();
    const Composite* d_comp = (const Composite*)(ws->dev_in + o_comp);
    DECODE_CK(cudaMemcpyAsync(ws->dev_in, ws->host, total_in, cudaMemcpyHostToDevice, st));
    DECODE_CK(cudaMemsetAsync(ws->zs, 0, (size_t)ztotal, st));
    DECODE_CK(cudaMemsetAsync(ws->sums, 0, sizeof(unsigned long long) * 2 * n, st));
    if (int rc = composite_launch(&cs, d_comp, (const PanelImg*)(ws->dev_in + o_pan), n, st, launches, err)) return rc;
    const unsigned bgrid = (unsigned)((total + 255) / 256);
    filter_kernel<<<dim3((unsigned)((max_pix + 255) / 256), n), 256, 0, st>>>(d_img, d_comp, cs.labels, ws->raw);
    runs_kernel<<<bgrid, 256, 0, st>>>(d_img, n, total, ws->raw, ws->counts);
    DECODE_CK(cudaGetLastError());
    if (int rc = exclusive_scan(&ws->tiles, ws->counts, total, ws->x, st, err)) return rc;
    runpos_kernel<<<bgrid, 256, 0, st>>>(d_img, n, total, ws->raw, ws->x, ws->runpos);
    parse_kernel<<<bgrid, 256, 0, st>>>(d_img, n, total, ws->raw, ws->x, ws->runpos, ws->tok, ws->counts);
    DECODE_CK(cudaGetLastError());
    if (int rc = exclusive_scan(&ws->tiles, ws->counts, total, ws->x, st, err)) return rc;
    compact_kernel<<<bgrid, 256, 0, st>>>(d_img, n, total, ws->tok, ws->x, ws->sym, ws->blks);
    histogram_kernel<<<(unsigned)nblk, 256, 0, st>>>(d_img, n, ws->x, ws->sym, ws->hist);
    trees_kernel<<<(unsigned)((nblk + 63) / 64), 64, 0, st>>>(d_img, n, nblk, ws->x, ws->hist, ws->blks);
    adler_kernel<<<dim3((unsigned)((max_n + ADLER_TILE - 1) / ADLER_TILE), n), 256, 0, st>>>(d_img, ws->raw, ws->sums);
    walk_kernel<<<1, 256, 0, st>>>(d_img, n, ws->blks, ws->sums, ws->zs, ws->out);
    emit_kernel<<<(unsigned)nblk, EMIT_THREADS, 0, st>>>(d_img, n, ws->blks, ws->sym, ws->raw, ws->out, ws->zs);
    DECODE_CK(cudaGetLastError());
    *launches += 16;
    DECODE_CK(cudaMemcpyAsync(ws->out_host, ws->out, sizeof(ImgOut) * n, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    const ImgOut* O = ws->out_host;
    for (int i = 0; i < n; i++) {
        if (O[i].zlen < 0) {  // the zcap bound does not hold: a defect, never expected
            *err = std::string(kCall) + ": frame " + std::to_string(i) + " exceeds the zlib stream's size bound";
            return -1;
        }
    }
    const long long total_file = O[n - 1].file0 + 8 + 25 + 12 * ((O[n - 1].zlen + IDAT_BYTES - 1) / IDAT_BYTES) + O[n - 1].zlen + 12;
    DECODE_CK(ws->file.grow((size_t)total_file));
    DECODE_CK(ws->result.grow((size_t)total_file));
    frame_kernel<<<(unsigned)O[0].chunks, FRAME_THREADS, 0, st>>>(d_img, n, ws->out, ws->zs, ws->file);
    DECODE_CK(cudaGetLastError());
    ++*launches;
    DECODE_CK(cudaMemcpyAsync(ws->result, ws->file, (size_t)total_file, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    for (int i = 0; i < n; i++) {
        uint8_t* f = ws->result + O[i].file0;
        static const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
        memcpy(f, kSig, 8);
        uint8_t* ihdr = f + 8;
        put_be32_host(ihdr + 8, (uint32_t)imgs[i].w);
        put_be32_host(ihdr + 12, (uint32_t)imgs[i].h);
        const uint8_t tail[5] = {8, 2, 0, 0, 0};
        memcpy(ihdr + 16, tail, 5);
        host_chunk(ihdr, "IHDR", 13);
        const long long size = 8 + 25 + 12 * ((O[i].zlen + IDAT_BYTES - 1) / IDAT_BYTES) + O[i].zlen + 12;
        host_chunk(f + size - 12, "IEND", 0);
        ws->res_off.push_back(O[i].file0);
        ws->res_len.push_back(size);
        nbytes[i] = size;
    }
    return 0;
}

}  // namespace smapb
