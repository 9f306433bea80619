// PNG decoding on the GPU, byte-identical to cv2.imdecode(buf, IMREAD_COLOR).
//
// Host: one bounds-checked chunk walk (png_parse) yields the geometry, the palette, the EXIF orientation and the IDAT
// chunks; everything it does not accept gets a status and is left to the caller's cv2 path.  It accepts every legal bit
// depth / colour type pair, interlace 0 and Adam7, PLTE, eXIf and ancillary chunks with a correct CRC; it refuses APNG,
// unknown critical chunks, a PLTE in a grey image, IDATs that are not consecutive, anything after the zlib stream's
// Adler-32 and a stream that inflates to more or fewer bytes than the scanlines need.  cv2 keeps 16-bit samples' high
// byte, drops alpha without compositing, ignores tRNS, gAMA, sBIT and bKGD, and reads a palette index past PLTE's
// entries as black; so does the colour kernel.
//
// Device: one launch per phase for the whole batch:
//   1. gather_kernel    one CTA per image copies its IDAT payloads into one contiguous zlib stream and checks each IDAT's
//                       CRC-32 (per-thread slice CRCs joined with the GF(2) shift x^(8n) mod P)
//   2. find_kernel      one thread per bit offset: could a dynamic DEFLATE block header start here (BTYPE 2, HLIT and HDIST
//                       <= 29, a complete code-length code, lengths that decode inside the header, a complete
//                       literal/length code with symbol 256)?  The block finder of parallel gzip decoders (Kerbiriou &
//                       Chikhi 2019, Knespel & Brunst 2023).
//   3. count_kernel     one thread per candidate decodes its block without writing: end bit, output length, validity;
//                       capped at COUNT_MAX_SYMBOLS symbols
//   4. chain_kernel     one thread per image follows the real blocks from the first one to the final one: a confirmed
//                       dynamic block jumps to its recorded end, a stored block by LEN, anything else (fixed Huffman, a
//                       dynamic block the finder missed or could not confirm) is decoded serially.  The running sum of
//                       the lengths is each block's output offset.  Correctness never rests on the finder: the chain only
//                       starts at the true first block and follows real block ends.
//   5. write_kernel     one thread per chained block decodes it again into uint16: 0..255 literals, 256 + i = byte i of
//                       the 32 KB window in front of the block (a match reaching before the block's first byte)
//   6. resolve_kernel   one CTA per image walks its blocks in order, replaces the window markers with the bytes already
//                       resolved, computes the Adler-32 and checks it
//   7. unfilter_kernel  one CTA per (image, Adam7 pass): a wavefront in which row r runs one unit behind row r - 1
//   8. colour_kernel    bit unpacking, palette, grey replication, high bytes, RGB -> BGR, Adam7 scatter, EXIF orientation
// Two valid streams that cv2 reads are refused on the device (SMAPB_JPEG_UNSUPPORTED and SMAPB_JPEG_CORRUPT) and left to
// cv2: one with more DEFLATE blocks than blk_cap = zlen / 8 + 64, the block records reserved per image (an exact bound, one
// block per 10 bits, would take 6.4 times the memory; a run of empty fixed blocks such as Z_PARTIAL_FLUSH writes reaches
// it), and one with a match that reaches past the window its zlib header's CINFO declares (zlib only refuses a distance
// past the bytes it holds, so whether cv2 reads it depends on the output buffers libpng hands to inflate).
// oracle/png_numpy.py restates the walk and the pixel rules, oracle/inflate_numpy.py the block structure and the finder.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/smap_b200.h"
#include "checksum.cuh"
#include "decode_host.h"
#include "orient.h"
#include "png.h"

namespace smapb {
namespace {

constexpr int COUNT_MAX_SYMBOLS = 1 << 16;  // a candidate that runs longer is left to the serial walk
constexpr int64_t MAX_STREAM_BYTES = 1 << 28;  // bit positions are 32-bit
constexpr int WINDOW = 32768;

struct DevPng {
    int h, w, depth, ctype, out_h, out_w, orientation;
    int chans, bpp, wsize, npass;
    int chunk0, nchunk;
    uint32_t zbits;            // zlib stream length in bits (the two header bytes included)
    int64_t zoff;              // the image's stream in the stream buffer (bytes, 16-aligned)
    int64_t raw_off, raw_len;  // its inflated scanlines in the raw / marker buffers
    int64_t blk_off;           // its block records
    int blk_cap;
    int pw[7], ph[7];
    int64_t prow[7], poff[7];  // bytes per row of each pass (the filter byte included), offset of the pass in raw
    uint8_t* out;
    uint8_t pal[768];          // zero-padded to 256 entries
};

struct DevChunk {
    int img;
    uint32_t len, crc;
    int64_t src;  // the chunk type's first byte in the staged input (the CRC covers type and payload)
    int64_t dst;  // its payload's first byte within the image's stream
};

struct DevBlock {
    uint32_t start, end;  // bits; end = the first bit after the block
    int out_off, out_len;
};

struct CountResult {
    uint32_t end;
    int out_len;
    int ok;
};

enum { ST_CAND = 0, ST_ONCHAIN = 1, ST_CONFIRMED = 2, ST_SERIAL = 3 };

// ---- host chunk walk -------------------------------------------------------------------------------------------------
inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

struct PngHeader {
    int w = 0, h = 0, depth = 0, ctype = 0, interlace = 0, orientation = 1, out_h = 0, out_w = 0, npal = 0, wsize = 0;
    uint8_t pal[768];
    std::vector<int64_t> idat;  // offsets of the IDAT chunks' type bytes
    std::vector<uint32_t> idat_len, idat_crc;
    int64_t zlen = 0;
};

bool legal_depth(int ctype, int depth) {
    switch (ctype) {
        case 0: return depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16;
        case 3: return depth == 1 || depth == 2 || depth == 4 || depth == 8;
        case 2: case 4: case 6: return depth == 8 || depth == 16;
        default: return false;
    }
}

int channels(int ctype) { return ctype == 2 ? 3 : ctype == 4 ? 2 : ctype == 6 ? 4 : 1; }

const int A7_YS[7] = {0, 0, 4, 0, 2, 0, 1}, A7_XS[7] = {0, 4, 0, 2, 0, 1, 0};
const int A7_DY[7] = {8, 8, 8, 4, 4, 2, 2}, A7_DX[7] = {8, 8, 4, 4, 2, 2, 1};

// Walks the chunks up to IEND.  Status SMAPB_JPEG_*: MALFORMED for data that is not a PNG or breaks its structure,
// CORRUPT for a chunk CRC or zlib header that is wrong, UNSUPPORTED for files that are valid but left to cv2, TOO_LARGE.
int png_parse(const uint8_t* d, int64_t n, PngHeader* H) {
    static const uint8_t SIG[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    if (!d || n < 8 || memcmp(d, SIG, 8) != 0) return SMAPB_JPEG_MALFORMED;
    memset(H->pal, 0, sizeof(H->pal));
    int64_t p = 8;
    bool ihdr = false, plte = false, exif = false, iend = false, idat_done = false;
    while (p < n) {
        if (n - p < 12) return SMAPB_JPEG_MALFORMED;
        const uint32_t len = be32(d + p);
        const uint8_t* t = d + p + 4;
        if (len > 0x7fffffffu || (int64_t)len > n - p - 12) return SMAPB_JPEG_MALFORMED;
        for (int k = 0; k < 4; k++)
            if (!((t[k] >= 'A' && t[k] <= 'Z') || (t[k] >= 'a' && t[k] <= 'z'))) return SMAPB_JPEG_MALFORMED;
        const uint8_t* s = t + 4;
        const uint32_t crc = be32(s + len);
        const bool is_idat = memcmp(t, "IDAT", 4) == 0;
        if (!ihdr && memcmp(t, "IHDR", 4) != 0) return SMAPB_JPEG_MALFORMED;
        if (!is_idat && crc32_host(t, 4 + (int64_t)len) != crc) return SMAPB_JPEG_CORRUPT;  // IDATs: on the device
        if (!H->idat.empty() && !is_idat) idat_done = true;
        if (memcmp(t, "IHDR", 4) == 0) {
            if (ihdr || len != 13) return SMAPB_JPEG_MALFORMED;
            ihdr = true;
            const uint32_t w = be32(s), h = be32(s + 4);
            H->depth = s[8], H->ctype = s[9], H->interlace = s[12];
            if (w == 0 || h == 0 || w > 0x7fffffffu || h > 0x7fffffffu || !legal_depth(H->ctype, H->depth) || s[10] != 0 ||
                s[11] != 0 || H->interlace > 1)
                return SMAPB_JPEG_MALFORMED;
            if ((uint64_t)w * h > (uint64_t)SMAPB_JPEG_MAX_PIXELS) return SMAPB_JPEG_TOO_LARGE;
            H->w = (int)w, H->h = (int)h;
        } else if (memcmp(t, "PLTE", 4) == 0) {
            if (plte || !H->idat.empty()) return SMAPB_JPEG_UNSUPPORTED;
            if (H->ctype == 0 || H->ctype == 4) return SMAPB_JPEG_UNSUPPORTED;  // cv2 warns and ignores it
            if (len == 0 || len % 3 || len > 768) return SMAPB_JPEG_MALFORMED;
            plte = true;
            if (H->ctype == 3) {
                H->npal = (int)len / 3;
                if (H->npal > (1 << H->depth)) return SMAPB_JPEG_UNSUPPORTED;
                memcpy(H->pal, s, len);
            }
        } else if (is_idat) {
            if (idat_done) return SMAPB_JPEG_UNSUPPORTED;  // IDATs must be consecutive
            if (H->ctype == 3 && !plte) return SMAPB_JPEG_MALFORMED;
            H->idat.push_back(p + 4);
            H->idat_len.push_back(len);
            H->idat_crc.push_back(crc);
            H->zlen += len;
        } else if (memcmp(t, "IEND", 4) == 0) {
            if (len != 0) return SMAPB_JPEG_MALFORMED;
            iend = true;
            break;
        } else if (memcmp(t, "eXIf", 4) == 0) {
            if (exif) return SMAPB_JPEG_UNSUPPORTED;
            exif = true;
            const int o = exif_tiff_orientation(s, len);
            if (o < 0) return SMAPB_JPEG_UNSUPPORTED;
            H->orientation = o;
        } else if (memcmp(t, "acTL", 4) == 0 || memcmp(t, "fcTL", 4) == 0 || memcmp(t, "fdAT", 4) == 0) {
            return SMAPB_JPEG_UNSUPPORTED;  // APNG
        } else if (!(t[0] & 0x20)) {
            return SMAPB_JPEG_UNSUPPORTED;  // an unknown critical chunk: cv2 refuses the file
        }
        p += 12 + (int64_t)len;
    }
    if (!ihdr || !iend || H->idat.empty()) return SMAPB_JPEG_MALFORMED;
    if (H->zlen > MAX_STREAM_BYTES) return SMAPB_JPEG_TOO_LARGE;
    // zlib header (its two bytes may lie in two IDATs)
    uint8_t zh[2];
    int got = 0;
    for (size_t c = 0; c < H->idat.size() && got < 2; c++)
        for (uint32_t k = 0; k < H->idat_len[c] && got < 2; k++) zh[got++] = d[H->idat[c] + 4 + k];
    if (got < 2) return SMAPB_JPEG_CORRUPT;
    if ((zh[0] & 15) != 8 || (zh[0] >> 4) > 7 || ((zh[0] << 8) | zh[1]) % 31 != 0) return SMAPB_JPEG_CORRUPT;
    if (zh[1] & 0x20) return SMAPB_JPEG_UNSUPPORTED;  // preset dictionary
    H->wsize = 1 << ((zh[0] >> 4) + 8);
    H->out_h = H->orientation >= 5 ? H->w : H->h;
    H->out_w = H->orientation >= 5 ? H->h : H->w;
    return SMAPB_JPEG_OK;
}

// ---- device: bits and Huffman codes ----------------------------------------------------------------------------------
// The 32 stream bits from bit `pos` on, first bit in bit 0.  The stream is padded with 16 zero bytes, so pos <= zbits reads
// inside the buffer.
__device__ __forceinline__ uint32_t peek32(const uint32_t* __restrict__ words, uint32_t pos) {
    return __funnelshift_r(words[pos >> 5], words[(pos >> 5) + 1], pos & 31);
}

constexpr int FAST_BITS = 9;

// Canonical Huffman code as zlib's inflate builds it: a 9-bit table for short codes (len << 9 | symbol, 0 = longer or
// unused), counts and the symbols in code order for the rest.
struct Huff {
    uint16_t fast[1 << FAST_BITS];
    uint16_t count[16];
    uint16_t sym[288];
};

// false where zlib's inflate_table fails: an over-subscribed code, or an incomplete one other than a single 1-bit code.
// A code with no symbols at all builds (every lookup fails).
__device__ bool huff_build(Huff& H, const uint8_t* lens, int n) {
    for (int l = 0; l < 16; l++) H.count[l] = 0;
    for (int s = 0; s < n; s++) H.count[lens[s]]++;
    H.count[0] = 0;
    int maxl = 0;
    for (int l = 1; l < 16; l++)
        if (H.count[l]) maxl = l;
    int left = 1;
    for (int l = 1; l < 16; l++) {
        left = (left << 1) - H.count[l];
        if (left < 0) return false;
    }
    if (left > 0 && maxl > 1) return false;
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + H.count[l];
    for (int s = 0; s < n; s++)
        if (lens[s]) H.sym[offs[lens[s]]++] = (uint16_t)s;
    for (int i = 0; i < (1 << FAST_BITS); i++) H.fast[i] = 0;
    int code = 0, k = 0;
    for (int l = 1; l <= FAST_BITS; l++) {
        for (int i = 0; i < H.count[l]; i++, k++, code++) {
            const int rev = __brev(code) >> (32 - l);
            for (int j = rev; j < (1 << FAST_BITS); j += 1 << l) H.fast[j] = (uint16_t)((l << 9) | H.sym[k]);
        }
        code <<= 1;
    }
    return true;
}

// Decodes one symbol from `bits`; -1 = no symbol of the code starts there.
__device__ __forceinline__ int huff_decode(const Huff& H, uint32_t bits, int* len) {
    const int e = H.fast[bits & ((1 << FAST_BITS) - 1)];
    if (e) {
        *len = e >> 9;
        return e & 511;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; l++) {
        code |= (bits >> (l - 1)) & 1;
        const int c = H.count[l];
        if (code - c < first) {
            *len = l;
            return H.sym[index + code - first];
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                     131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                     2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// Reads the code lengths of a dynamic block whose 3 header bits start at `pos`; on success *pos is the first bit of the
// block's data and lens[0..nlen + ndist) holds the lengths.  `strict` adds the finder's test that the literal/length code
// is complete (zlib also accepts an incomplete one made of a single 1-bit code).  false = not a valid header for zlib.
__device__ bool dyn_header(const uint32_t* __restrict__ words, uint32_t zbits, uint32_t* pos, uint8_t* lens, int* nlen,
                           int* ndist, bool strict) {
    uint32_t p = *pos;
    if (p + 17 > zbits) return false;
    const uint32_t v = peek32(words, p);
    if (((v >> 1) & 3) != 2) return false;
    const int hlit = (v >> 3) & 31, hdist = (v >> 8) & 31, hclen = ((v >> 13) & 15) + 4;
    if (hlit > 29 || hdist > 29) return false;
    p += 17;
    if (p + 3 * hclen > zbits) return false;
    uint8_t cl[19];
    for (int i = 0; i < 19; i++) cl[i] = 0;
    for (int i = 0; i < hclen; i++) cl[c_clorder[i]] = (peek32(words, p + 3 * i)) & 7;
    p += 3 * hclen;
    // the code-length code must be complete (zlib refuses an incomplete one): Kraft sum over 7-bit codes = 128
    int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 19; i++) cnt[cl[i]]++;
    int kraft = 0;
    for (int l = 1; l < 8; l++) kraft += cnt[l] << (7 - l);
    if (kraft != 128) return false;
    uint8_t tab[128];  // 7-bit lookup: len << 5 | symbol
    {
        int offs[8], code = 0;
        uint8_t syms[19];
        offs[1] = 0;
        for (int l = 1; l < 7; l++) offs[l + 1] = offs[l] + cnt[l];
        for (int s = 0; s < 19; s++)
            if (cl[s]) syms[offs[cl[s]]++] = (uint8_t)s;
        int k = 0;
        for (int l = 1; l < 8; l++) {
            for (int i = 0; i < cnt[l]; i++, k++, code++) {
                const int rev = __brev(code) >> (32 - l);
                for (int j = rev; j < 128; j += 1 << l) tab[j] = (uint8_t)((l << 5) | syms[k]);
            }
            code <<= 1;
        }
    }
    const int nl = hlit + 257, nd = hdist + 1, total = nl + nd;
    int i = 0;
    while (i < total) {
        if (p > zbits) return false;
        const uint32_t b = peek32(words, p);
        const int e = tab[b & 127], l = e >> 5, s = e & 31;
        p += l;
        if (s < 16) {
            lens[i++] = (uint8_t)s;
            continue;
        }
        int rep, val = 0;
        if (s == 16) {
            if (i == 0) return false;
            val = lens[i - 1], rep = 3 + ((b >> l) & 3), p += 2;
        } else if (s == 17) {
            rep = 3 + ((b >> l) & 7), p += 3;
        } else {
            rep = 11 + ((b >> l) & 127), p += 7;
        }
        if (i + rep > total) return false;
        while (rep--) lens[i++] = (uint8_t)val;
    }
    if (p > zbits || lens[256] == 0) return false;
    if (strict) {
        int kr = 0;  // in units of 2^-15
        for (int s = 0; s < nl; s++)
            if (lens[s]) kr += 1 << (15 - lens[s]);
        if (kr != 1 << 15) return false;
    }
    *pos = p, *nlen = nl, *ndist = nd;
    return true;
}

enum { INF_OK = 0, INF_BAD = 1, INF_CAP = 2 };

// Decodes one fixed (type 1) or dynamic (type 2) block from its header bit `start`.  COUNT: *out_len = bytes it yields,
// nothing written, more than max_syms symbols = INF_CAP.  WRITE: the block's bytes go to blk[0..out_len) as uint16, a
// match reaching `blk_base` bytes or more back (before the block) as the window marker 256 + i; a match reaching before
// the stream's first byte is INF_BAD.  Either way: INF_BAD where zlib fails (an unused code, a length or distance symbol
// outside the tables, a distance past the header's window, data past the stream's end) or where the block yields more
// than out_cap bytes.
template <bool WRITE>
__device__ int inflate_block(const uint32_t* __restrict__ words, uint32_t zbits, uint32_t start, int type, int wsize,
                             int64_t out_cap, int max_syms, uint16_t* blk, int64_t blk_base, uint32_t* end, int* final,
                             int* out_len, Huff& L, Huff& D) {
    uint32_t pos = start;
    if (pos + 3 > zbits) return INF_BAD;
    *final = peek32(words, pos) & 1;
    uint8_t lens[320];
    if (type == 2) {
        int nl, nd;
        if (!dyn_header(words, zbits, &pos, lens, &nl, &nd, false)) return INF_BAD;
        if (!huff_build(L, lens, nl) || !huff_build(D, lens + nl, nd)) return INF_BAD;
    } else {
        pos += 3;
        for (int s = 0; s < 288; s++) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        for (int s = 0; s < 32; s++) lens[288 + s] = 5;  // 30 and 31 complete the code; decoding them is an error
        huff_build(L, lens, 288);
        huff_build(D, lens + 288, 32);
    }
    int64_t n = 0;
    int syms = 0;
    for (;;) {
        if (pos > zbits) return INF_BAD;
        uint32_t b = peek32(words, pos);
        int l;
        int s = huff_decode(L, b, &l);
        if (s < 0) return INF_BAD;
        pos += l;
        if (s == 256) break;
        if (!WRITE && ++syms > max_syms) return INF_CAP;
        if (s < 256) {
            if (n >= out_cap) return INF_BAD;
            if (WRITE) blk[n] = (uint16_t)s;
            n++;
            continue;
        }
        s -= 257;
        if (s >= 29) return INF_BAD;
        const int le = c_lext[s];
        const int len = c_lbase[s] + (int)((b >> l) & ((1u << le) - 1));
        pos += le;
        if (pos > zbits) return INF_BAD;
        b = peek32(words, pos);
        const int ds = huff_decode(D, b, &l);
        if (ds < 0 || ds >= 30) return INF_BAD;
        pos += l;
        const int de = c_dext[ds];
        const int dist = c_dbase[ds] + (int)((b >> l) & ((1u << de) - 1));
        pos += de;
        if (dist > wsize || n + len > out_cap) return INF_BAD;
        if (WRITE) {
            if (blk_base + n - dist < 0) return INF_BAD;  // before the stream's first byte
            const int64_t src = n - dist;                 // relative to the block: < 0 = in the window in front of it
            for (int k = 0; k < len; k += 8) {
                uint16_t t[8];
                const int c = min(8, len - k);
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (j < c) {
                        const int64_t q = src + (dist >= len ? k + j : (k + j) % dist);
                        t[j] = q < 0 ? (uint16_t)(256 + WINDOW + q) : blk[q];
                    }
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (j < c) blk[n + k + j] = t[j];
            }
        }
        n += len;
    }
    if (pos > zbits) return INF_BAD;
    *end = pos;
    *out_len = (int)n;
    return INF_OK;
}

// A stored block at `start`: its payload's first byte and length; false = LEN / NLEN disagree or it runs past the stream.
__device__ bool stored_block(const uint32_t* __restrict__ words, uint32_t zbits, uint32_t start, uint32_t* data, int* len) {
    const uint32_t p = (start + 3 + 7) & ~7u;
    if (p + 32 > zbits) return false;
    const uint32_t v = peek32(words, p);
    if ((v & 0xffff) != (~v >> 16)) return false;
    *len = (int)(v & 0xffff);
    *data = p + 32;
    return (uint64_t)*data + 8ull * *len <= zbits;
}

__device__ __forceinline__ void set_status(int* status, int img, int s) { atomicCAS(&status[img], SMAPB_JPEG_OK, s); }

// ---- 1. gather + IDAT CRCs -------------------------------------------------------------------------------------------
constexpr int GATHER_THREADS = 512;

__global__ void __launch_bounds__(GATHER_THREADS) gather_kernel(const DevPng* __restrict__ imgs, const DevChunk* __restrict__ chunks,
                                                                const uint8_t* __restrict__ in, uint8_t* __restrict__ stream,
                                                                int* __restrict__ status) {
    __shared__ uint32_t T[256], x2n[32], red[GATHER_THREADS / 32];
    const DevPng& I = imgs[blockIdx.x];
    const int tid = threadIdx.x;
    crc_tables(T, x2n);
    uint8_t* zs = stream + I.zoff;
    const int64_t zlen = I.zbits / 8;
    for (int i = tid; i < 16; i += blockDim.x) zs[zlen + i] = 0;
    for (int c = 0; c < I.nchunk; c++) {
        const DevChunk C = chunks[I.chunk0 + c];
        const uint8_t* src = in + C.src;
        for (uint32_t j = tid; j < C.len; j += blockDim.x) zs[C.dst + j] = src[4 + j];
        // CRC over type + payload
        const uint64_t L = 4ull + C.len;
        uint32_t r = crc_slice(T, x2n, L, [&](uint64_t j) { return src[j]; });
        for (int o = 16; o; o >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, o);
        if ((tid & 31) == 0) red[tid >> 5] = r;
        __syncthreads();
        if (tid == 0) {
            uint32_t t = 0;
            for (int w = 0; w < (int)(blockDim.x / 32); w++) t ^= red[w];
            if (crc_finish(x2n, L, t) != C.crc) set_status(status, blockIdx.x, SMAPB_JPEG_CORRUPT);
        }
        __syncthreads();
    }
}

// ---- 2. block finder -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long cand_key(int img, uint32_t bit) { return ((unsigned long long)img << 32 | bit) + 1; }

__device__ __forceinline__ uint32_t hash_slot(unsigned long long key, uint32_t mask) {
    return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask;
}

__global__ void __launch_bounds__(256) find_kernel(const DevPng* __restrict__ imgs, const uint8_t* __restrict__ stream,
                                                   const int* __restrict__ status, unsigned long long* __restrict__ cand,
                                                   int cand_cap, unsigned long long* __restrict__ hkey, int* __restrict__ hval,
                                                   uint32_t hmask, int* __restrict__ stats) {
    const int img = blockIdx.y;
    const DevPng& I = imgs[img];
    const uint32_t bit = (uint32_t)blockIdx.x * blockDim.x + threadIdx.x + 16;  // the first block starts after the header
    if (bit + 17 > I.zbits || status[img] != SMAPB_JPEG_OK) return;
    const uint32_t* words = (const uint32_t*)(stream + I.zoff);
    const uint32_t v = peek32(words, bit);
    if (((v >> 1) & 3) != 2 || ((v >> 3) & 31) > 29 || ((v >> 8) & 31) > 29) return;
    uint8_t lens[320];
    uint32_t p = bit;
    int nl, nd;
    if (!dyn_header(words, I.zbits, &p, lens, &nl, &nd, true)) return;
    const int i = atomicAdd(&stats[ST_CAND], 1);
    if (i >= cand_cap) return;  // the serial walk decodes what does not fit
    const unsigned long long key = cand_key(img, bit);
    cand[i] = key;
    for (uint32_t h = hash_slot(key, hmask);; h = (h + 1) & hmask) {
        if (atomicCAS(&hkey[h], 0ull, key) == 0ull) {
            hval[h] = i;
            break;
        }
    }
}

// ---- 3. speculative count pass ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) count_kernel(const DevPng* __restrict__ imgs, const uint8_t* __restrict__ stream,
                                                   const unsigned long long* __restrict__ cand, const int* __restrict__ stats,
                                                   int cand_cap, CountResult* __restrict__ res) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(stats[ST_CAND], cand_cap)) return;
    const unsigned long long key = cand[i] - 1;
    const DevPng& I = imgs[key >> 32];
    Huff L, D;
    CountResult r;
    int final;
    r.ok = inflate_block<false>((const uint32_t*)(stream + I.zoff), I.zbits, (uint32_t)key, 2, I.wsize, I.raw_len,
                                COUNT_MAX_SYMBOLS, nullptr, 0, &r.end, &final, &r.out_len, L, D) == INF_OK;
    res[i] = r;
}

// ---- 4. chain walk ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) chain_kernel(const DevPng* __restrict__ imgs, int m, const uint8_t* __restrict__ stream,
                                                   const unsigned long long* __restrict__ hkey, const int* __restrict__ hval,
                                                   uint32_t hmask, const CountResult* __restrict__ res, DevBlock* __restrict__ blocks,
                                                   int* __restrict__ nblk, uint32_t* __restrict__ adler, int* __restrict__ status,
                                                   int* __restrict__ stats) {
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= m) return;
    nblk[img] = 0;
    const DevPng& I = imgs[img];
    if (status[img] != SMAPB_JPEG_OK) return;
    const uint32_t* words = (const uint32_t*)(stream + I.zoff);
    DevBlock* B = blocks + I.blk_off;
    Huff L, D;
    uint32_t pos = 16;
    int64_t n = 0;
    int k = 0, onchain = 0, confirmed = 0, serial = 0, bad = 0;
    for (;;) {
        if (k == I.blk_cap) {
            bad = SMAPB_JPEG_UNSUPPORTED;
            break;
        }
        if (pos + 3 > I.zbits) {
            bad = SMAPB_JPEG_CORRUPT;
            break;
        }
        const uint32_t v = peek32(words, pos);
        const int final = v & 1, type = (v >> 1) & 3;
        uint32_t end = 0;
        int len = 0;
        if (type == 0) {
            uint32_t data;
            if (!stored_block(words, I.zbits, pos, &data, &len)) {
                bad = SMAPB_JPEG_CORRUPT;
                break;
            }
            end = data + 8u * len;
            serial++;
        } else if (type == 3) {
            bad = SMAPB_JPEG_CORRUPT;
            break;
        } else {
            bool done = false;
            if (type == 2) {
                const unsigned long long key = cand_key(img, pos);
                for (uint32_t h = hash_slot(key, hmask); hkey[h]; h = (h + 1) & hmask)
                    if (hkey[h] == key) {
                        const CountResult r = res[hval[h]];
                        onchain++;
                        if (r.ok) end = r.end, len = r.out_len, done = true, confirmed++;
                        break;
                    }
            }
            if (!done) {
                int f;
                if (inflate_block<false>(words, I.zbits, pos, type, I.wsize, I.raw_len, INT_MAX, nullptr, 0, &end, &f, &len, L,
                                         D) != INF_OK) {
                    bad = SMAPB_JPEG_CORRUPT;
                    break;
                }
                serial++;
            }
        }
        if (n + len > I.raw_len) {  // more data than the scanlines need
            bad = SMAPB_JPEG_UNSUPPORTED;
            break;
        }
        B[k].start = pos, B[k].end = end, B[k].out_off = (int)n, B[k].out_len = len;
        n += len, k++;
        pos = end;
        if (final) break;
    }
    atomicAdd(&stats[ST_ONCHAIN], onchain);
    atomicAdd(&stats[ST_CONFIRMED], confirmed);
    atomicAdd(&stats[ST_SERIAL], serial);
    if (!bad) {
        pos = (pos + 7) & ~7u;
        if (pos + 32 > I.zbits || n != I.raw_len) bad = SMAPB_JPEG_CORRUPT;  // no Adler-32, or not enough image data
        else if (pos + 32 != I.zbits) bad = SMAPB_JPEG_UNSUPPORTED;        // bytes after the zlib stream
    }
    if (bad) {
        set_status(status, img, bad);
        return;
    }
    const uint32_t a = __byte_perm(peek32(words, pos), 0, 0x0123);  // big-endian
    adler[img] = a;
    nblk[img] = k;
}

// ---- 5. write pass ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) write_kernel(const DevPng* __restrict__ imgs, const uint8_t* __restrict__ stream,
                                                   const DevBlock* __restrict__ blocks, const int* __restrict__ nblk,
                                                   uint16_t* __restrict__ marks, int* __restrict__ status) {
    const int img = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nblk[img] || status[img] != SMAPB_JPEG_OK) return;
    const DevPng& I = imgs[img];
    const DevBlock Bk = blocks[I.blk_off + k];
    const uint32_t* words = (const uint32_t*)(stream + I.zoff);
    uint16_t* out = marks + I.raw_off + Bk.out_off;
    const int type = (peek32(words, Bk.start) >> 1) & 3;
    if (type == 0) {
        uint32_t data;
        int len;
        stored_block(words, I.zbits, Bk.start, &data, &len);
        const uint8_t* s = stream + I.zoff + data / 8;
        for (int j = 0; j < len; j++) out[j] = s[j];
        return;
    }
    Huff L, D;
    uint32_t end;
    int final, len;
    if (inflate_block<true>(words, I.zbits, Bk.start, type, I.wsize, Bk.out_len, INT_MAX, out, Bk.out_off, &end, &final, &len, L,
                            D) != INF_OK ||
        len != Bk.out_len || end != Bk.end)
        set_status(status, img, SMAPB_JPEG_CORRUPT);
}

// ---- 6. resolve + Adler-32 -------------------------------------------------------------------------------------------
constexpr int RESOLVE_THREADS = 1024;

__global__ void __launch_bounds__(RESOLVE_THREADS) resolve_kernel(const DevPng* __restrict__ imgs, const DevBlock* __restrict__ blocks,
                                                                  const int* __restrict__ nblk, const uint16_t* __restrict__ marks,
                                                                  uint8_t* __restrict__ raw, const uint32_t* __restrict__ adler,
                                                                  int* __restrict__ status) {
    __shared__ unsigned long long red[2][RESOLVE_THREADS / 32];
    const int img = blockIdx.x;
    const DevPng& I = imgs[img];
    if (status[img] != SMAPB_JPEG_OK) return;
    const uint16_t* mk = marks + I.raw_off;
    uint8_t* r = raw + I.raw_off;
    const int64_t N = I.raw_len;
    unsigned long long s1 = 0, s2 = 0;  // sum of bytes, sum of (N - i) * byte
    for (int k = 0; k < nblk[img]; k++) {
        const DevBlock Bk = blocks[I.blk_off + k];
        const int64_t base = Bk.out_off, win = base - WINDOW;
        for (int j0 = 0; j0 < Bk.out_len; j0 += 4 * RESOLVE_THREADS) {
            uint16_t v[4];
            uint8_t o[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int j = j0 + u * RESOLVE_THREADS + threadIdx.x;
                v[u] = j < Bk.out_len ? mk[base + j] : 0;
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int64_t q = win + (v[u] - 256);
                o[u] = v[u] < 256 ? (uint8_t)v[u] : q >= 0 ? r[q] : 0;  // q < 0 was refused by the write pass
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int j = j0 + u * RESOLVE_THREADS + threadIdx.x;
                if (j < Bk.out_len) {
                    r[base + j] = o[u];
                    s1 += o[u];
                    s2 += (unsigned long long)(N - (base + j)) * o[u];
                }
            }
        }
        s1 %= ADLER_MOD, s2 %= ADLER_MOD;
        __syncthreads();  // the next block reads these bytes
    }
    for (int o = 16; o; o >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, o), s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    if ((threadIdx.x & 31) == 0) red[0][threadIdx.x >> 5] = s1, red[1][threadIdx.x >> 5] = s2;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long a = 1, b = N % ADLER_MOD;
        for (int w = 0; w < RESOLVE_THREADS / 32; w++) a += red[0][w], b += red[1][w];
        if ((uint32_t)((b % ADLER_MOD) << 16 | (a % ADLER_MOD)) != adler[img]) set_status(status, img, SMAPB_JPEG_CORRUPT);
    }
}

// ---- 7. unfilter -----------------------------------------------------------------------------------------------------
// One CTA per (pass, image), in place: row r handles its bytes in units of 8 pixels (8 bytes below 8 bits per pixel), unit
// u at step r + u, so every unit finds the unit above and the one to its left done.  Rows go in groups of the CTA size.
constexpr int UNFILTER_THREADS = 1024;

__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

__global__ void __launch_bounds__(UNFILTER_THREADS) unfilter_kernel(const DevPng* __restrict__ imgs, uint8_t* __restrict__ raw,
                                                                    int* __restrict__ status) {
    const int img = blockIdx.y, pass = blockIdx.x;
    const DevPng& I = imgs[img];
    if (pass >= I.npass || status[img] != SMAPB_JPEG_OK) return;
    const int rows = I.ph[pass];
    if (rows == 0 || I.pw[pass] == 0) return;
    const int64_t stride = I.prow[pass], rb = stride - 1;
    const int bpp = I.bpp, unit = 8 * bpp;
    const int nunit = (int)((rb + unit - 1) / unit);
    uint8_t* base = raw + I.raw_off + I.poff[pass];
    __shared__ int bad;
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    for (int r0 = 0; r0 < rows; r0 += UNFILTER_THREADS) {
        const int r = r0 + threadIdx.x;
        const int nr = min(UNFILTER_THREADS, rows - r0);
        uint8_t* cur = base + (int64_t)r * stride;
        const uint8_t* prev = cur - stride;
        const int f = r < rows ? cur[0] : 0;
        if (f > 4) bad = 1;
        cur++, prev++;
        for (int s = 0; s < nunit + nr - 1; s++) {
            const int u = s - threadIdx.x;
            if (r < rows && u >= 0 && u < nunit && f != 0) {
                const int64_t a0 = (int64_t)u * unit, a1 = rb < a0 + unit ? rb : a0 + unit;
                for (int64_t i = a0; i < a1; i++) {
                    const int a = i >= bpp ? cur[i - bpp] : 0;
                    const int b = r > 0 ? prev[i] : 0;
                    const int c = r > 0 && i >= bpp ? prev[i - bpp] : 0;
                    const int x = cur[i];
                    cur[i] = (uint8_t)(f == 1 ? x + a : f == 2 ? x + b : f == 3 ? x + ((a + b) >> 1) : x + paeth(a, b, c));
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0 && bad) set_status(status, img, SMAPB_JPEG_CORRUPT);
}

// ---- 8. colour, Adam7 scatter, orientation ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colour_kernel(const DevPng* __restrict__ imgs, const uint8_t* __restrict__ raw,
                                                     const int* __restrict__ status) {
    const DevPng& I = imgs[blockIdx.y];
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)I.h * I.w || status[blockIdx.y] != SMAPB_JPEG_OK) return;
    const int y = (int)(t / I.w), x = (int)(t % I.w);
    int p = 0, py = y, px = x;
    if (I.npass == 7) {
        const int a7y[7] = {0, 0, 4, 0, 2, 0, 1}, a7x[7] = {0, 4, 0, 2, 0, 1, 0};
        const int a7dy[7] = {8, 8, 8, 4, 4, 2, 2}, a7dx[7] = {8, 8, 4, 4, 2, 2, 1};
        for (p = 0; p < 7; p++)
            if (y % a7dy[p] == a7y[p] && x % a7dx[p] == a7x[p]) break;
        py = y / a7dy[p], px = x / a7dx[p];
    }
    const uint8_t* row = raw + I.raw_off + I.poff[p] + (int64_t)py * I.prow[p] + 1;
    int r, g, b;
    if (I.depth < 8) {
        const int64_t bit = (int64_t)px * I.depth;
        const int v = (row[bit >> 3] >> (8 - I.depth - (int)(bit & 7))) & ((1 << I.depth) - 1);
        if (I.ctype == 3) {
            r = I.pal[3 * v], g = I.pal[3 * v + 1], b = I.pal[3 * v + 2];
        } else {
            r = g = b = v * 255 / ((1 << I.depth) - 1);
        }
    } else {
        const int sh = I.depth == 16 ? 1 : 0;  // 16-bit samples: the high (first) byte
        const uint8_t* s = row + (((int64_t)px * I.chans) << sh);
        if (I.ctype == 3) {
            r = I.pal[3 * s[0]], g = I.pal[3 * s[0] + 1], b = I.pal[3 * s[0] + 2];
        } else if (I.ctype == 0 || I.ctype == 4) {
            r = g = b = s[0];
        } else {
            r = s[0], g = s[1 << sh], b = s[2 << sh];
        }
    }
    int oy, ox;
    orient_store_pos(I.orientation, I.h, I.w, y, x, &oy, &ox);
    uint8_t* o = I.out + ((int64_t)oy * I.out_w + ox) * 3;
    o[0] = (uint8_t)b, o[1] = (uint8_t)g, o[2] = (uint8_t)r;
}

}  // namespace

// staging: descriptors and IDAT regions; small: stats[4] | status[m] | nblk[m] | adler[m]
struct PngWorkspace {
    PinnedBuffer<uint8_t> host;
    DeviceBuffer<uint8_t> dev_in;
    DeviceBuffer<int> small;
    PinnedBuffer<int> small_host;
    DeviceBuffer<uint8_t> stream;
    DeviceBuffer<unsigned long long> cand;
    DeviceBuffer<CountResult> res;
    DeviceBuffer<unsigned long long> hkey;
    DeviceBuffer<int> hval;
    DeviceBuffer<DevBlock> blocks;
    DeviceBuffer<uint16_t> marks;
    DeviceBuffer<uint8_t> raw;
    int64_t stats[4] = {0, 0, 0, 0};
};

PngWorkspace* png_workspace_create() { return new PngWorkspace(); }

void png_workspace_destroy(PngWorkspace* ws) { delete ws; }

void png_last_stats(const PngWorkspace* ws, int64_t out[4]) {
    for (int i = 0; i < 4; i++) out[i] = ws ? ws->stats[i] : 0;
}

int png_decode(PngWorkspace* ws, int n, const uint8_t* const* png, const int64_t* nbytes, uint8_t* const* bgr, int* status,
               cudaStream_t st, int64_t* launches, std::string* err) {
    for (int i = 0; i < 4; i++) ws->stats[i] = 0;
    std::vector<PngHeader> H;
    std::vector<int> idx;
    const int m = decode_preamble("smapb_decode_png", n, png, nbytes, bgr, status, st, png_parse, &H, &idx, err);
    if (m <= 0) return m;
    std::vector<DevPng> imgs(m);
    std::vector<DevChunk> chunks;
    int64_t in_total = 0, z_total = 0, raw_total = 0, blk_total = 0, max_px = 0;
    uint32_t max_zbits = 0;
    std::vector<int64_t> in_off(m), in_len(m);
    for (int k = 0; k < m; k++) {
        const PngHeader& h = H[idx[k]];
        DevPng& I = imgs[k];
        memset(&I, 0, sizeof(I));
        I.h = h.h, I.w = h.w, I.depth = h.depth, I.ctype = h.ctype, I.out_h = h.out_h, I.out_w = h.out_w;
        I.orientation = h.orientation, I.chans = channels(h.ctype), I.wsize = h.wsize;
        I.bpp = std::max(1, I.chans * h.depth / 8);
        I.npass = h.interlace ? 7 : 1;
        int64_t off = 0;
        for (int p = 0; p < I.npass; p++) {
            if (h.interlace) {
                I.pw[p] = (h.w - A7_XS[p] + A7_DX[p] - 1) / A7_DX[p];
                I.ph[p] = (h.h - A7_YS[p] + A7_DY[p] - 1) / A7_DY[p];
                if (I.pw[p] <= 0 || I.ph[p] <= 0) I.pw[p] = I.ph[p] = 0;
            } else {
                I.pw[p] = h.w, I.ph[p] = h.h;
            }
            I.prow[p] = 1 + ((int64_t)I.pw[p] * I.chans * h.depth + 7) / 8;
            I.poff[p] = off;
            off += I.pw[p] ? I.prow[p] * I.ph[p] : 0;
        }
        I.raw_len = off, I.raw_off = raw_total;
        raw_total += align_up(off, 16);
        I.zbits = (uint32_t)(h.zlen * 8);
        I.zoff = z_total;
        z_total += align_up(h.zlen + 16, 16);
        I.blk_cap = (int)std::min<int64_t>(h.zlen / 8 + 64, 1 << 30);
        I.blk_off = blk_total;
        blk_total += I.blk_cap;
        memcpy(I.pal, h.pal, sizeof(I.pal));
        I.out = bgr[idx[k]];
        // the staged region runs from the first IDAT's type to the last IDAT's CRC
        in_off[k] = in_total;
        const int64_t first = h.idat.front(), last = h.idat.back() + 4 + h.idat_len.back() + 4;
        in_len[k] = last - first;
        I.chunk0 = (int)chunks.size(), I.nchunk = (int)h.idat.size();
        int64_t dst = 0;
        for (size_t c = 0; c < h.idat.size(); c++) {
            DevChunk C;
            C.img = k, C.len = h.idat_len[c], C.crc = h.idat_crc[c], C.src = in_total + (h.idat[c] - first), C.dst = dst;
            dst += C.len;
            chunks.push_back(C);
        }
        in_total += align_up(in_len[k], 16);
        max_zbits = std::max(max_zbits, I.zbits);
        max_px = std::max(max_px, (int64_t)h.h * h.w);
    }
    const int cand_cap = (int)std::min<int64_t>(z_total / 64 + 4096, 1 << 26);
    uint32_t hsize = 1;
    while (hsize < 2u * cand_cap) hsize <<= 1;
    // staging layout: images | chunks | IDAT regions
    const size_t o_img = 0, o_chunk = align_up(sizeof(DevPng) * m, 256), o_in = align_up(o_chunk + sizeof(DevChunk) * chunks.size(), 256),
                 total = o_in + in_total;
    DECODE_CK(ws->host.grow(total));
    DECODE_CK(cudaStreamSynchronize(st));  // the staging area and the workspace may still be in use by the previous call
    memcpy(ws->host + o_img, imgs.data(), sizeof(DevPng) * m);
    memcpy(ws->host + o_chunk, chunks.data(), sizeof(DevChunk) * chunks.size());
    for (int k = 0; k < m; k++) memcpy(ws->host + o_in + in_off[k], png[idx[k]] + H[idx[k]].idat.front(), in_len[k]);
    const size_t nsmall = 4 + 3 * (size_t)m;
    DECODE_CK(ws->dev_in.grow(total));
    DECODE_CK(ws->stream.grow((size_t)z_total));
    DECODE_CK(ws->cand.grow((size_t)cand_cap));
    DECODE_CK(ws->res.grow((size_t)cand_cap));
    DECODE_CK(ws->hkey.grow((size_t)hsize));
    DECODE_CK(ws->hval.grow((size_t)hsize));
    DECODE_CK(ws->blocks.grow((size_t)blk_total));
    DECODE_CK(ws->marks.grow((size_t)raw_total));
    DECODE_CK(ws->raw.grow((size_t)raw_total));
    DECODE_CK(ws->small.grow(nsmall));
    DECODE_CK(ws->small_host.grow(nsmall));
    const DevPng* d_img = (const DevPng*)(ws->dev_in + o_img);
    const DevChunk* d_chunk = (const DevChunk*)(ws->dev_in + o_chunk);
    const uint8_t* d_in = ws->dev_in + o_in;
    int* d_stats = ws->small;
    int* d_status = ws->small + 4;
    int* d_nblk = d_status + m;
    uint32_t* d_adler = (uint32_t*)(d_nblk + m);
    int* hs = ws->small_host;
    for (int i = 0; i < 4; i++) hs[i] = 0;
    for (int k = 0; k < m; k++) hs[4 + k] = SMAPB_JPEG_OK;
    DECODE_CK(cudaMemcpyAsync(ws->dev_in, ws->host, total, cudaMemcpyHostToDevice, st));
    DECODE_CK(cudaMemcpyAsync(ws->small, hs, sizeof(int) * (4 + m), cudaMemcpyHostToDevice, st));
    DECODE_CK(cudaMemsetAsync(ws->hkey, 0, sizeof(unsigned long long) * hsize, st));
    gather_kernel<<<m, GATHER_THREADS, 0, st>>>(d_img, d_chunk, d_in, ws->stream, d_status);
    find_kernel<<<dim3((max_zbits + 255) / 256, m), 256, 0, st>>>(d_img, ws->stream, d_status, ws->cand, cand_cap, ws->hkey, ws->hval,
                                                                  hsize - 1, d_stats);
    count_kernel<<<(cand_cap + 63) / 64, 64, 0, st>>>(d_img, ws->stream, ws->cand, d_stats, cand_cap, ws->res);
    chain_kernel<<<(m + 31) / 32, 32, 0, st>>>(d_img, m, ws->stream, ws->hkey, ws->hval, hsize - 1, ws->res, ws->blocks, d_nblk,
                                               d_adler, d_status, d_stats);
    DECODE_CK(cudaGetLastError());
    *launches += 4;
    DECODE_CK(cudaMemcpyAsync(hs + 4 + m, d_nblk, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    int max_blk = 0;
    for (int k = 0; k < m; k++) max_blk = std::max(max_blk, hs[4 + m + k]);
    if (max_blk > 0) {
        write_kernel<<<dim3((max_blk + 63) / 64, m), 64, 0, st>>>(d_img, ws->stream, ws->blocks, d_nblk, ws->marks, d_status);
        resolve_kernel<<<m, RESOLVE_THREADS, 0, st>>>(d_img, ws->blocks, d_nblk, ws->marks, ws->raw, d_adler, d_status);
        unfilter_kernel<<<dim3(7, m), UNFILTER_THREADS, 0, st>>>(d_img, ws->raw, d_status);
        colour_kernel<<<dim3((unsigned)((max_px + 255) / 256), m), 256, 0, st>>>(d_img, ws->raw, d_status);
        DECODE_CK(cudaGetLastError());
        *launches += 4;
    }
    DECODE_CK(cudaMemcpyAsync(hs, ws->small, sizeof(int) * (4 + m), cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    ws->stats[0] = hs[ST_CAND];
    ws->stats[1] = hs[ST_CAND] - hs[ST_ONCHAIN];
    ws->stats[2] = hs[ST_CONFIRMED];
    ws->stats[3] = hs[ST_SERIAL];
    for (int k = 0; k < m; k++) status[idx[k]] = hs[4 + k];
    return 0;
}

}  // namespace smapb

extern "C" {
#pragma GCC visibility push(default)
int smapb_png_info(const uint8_t* data, int64_t nbytes, int* h, int* w, int* orientation, int* status) {
    if (!status) return -1;
    smapb::PngHeader H;
    return smapb::report_info(smapb::png_parse(data, nbytes, &H), H, status, h, w, orientation);
}
#pragma GCC visibility pop
}
