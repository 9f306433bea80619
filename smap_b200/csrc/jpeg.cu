// Huffman, 8-bit JPEG decoding on the GPU, byte-identical to cv2.imread(path, IMREAD_COLOR).
//
// Host: one bounds-checked marker walk (jpeg_parse) yields the frame (geometry, quantisers, EXIF orientation) and one
// ScanSpec per scan (the tables in force at its SOS, its band, its restart segments); anything it does not accept gets a
// status and is left to the caller's cv2 path.  Without SMAPB_JPEG_SCANS it accepts baseline files only: one interleaved
// sequential scan (SOF0/SOF1) of every component, then EOI.  With it, it also accepts sequential files with several scans
// and progressive Huffman files (SOF2): it walks every scan up to EOI, checks the progression as libjpeg does, latches each
// component's quantiser at its first scan, refuses what libjpeg-turbo would smooth (coefficients 1..9 not fully refined)
// and caps the scans at 64.
//
// Device: the coefficient buffer is zeroed once, then the scans run in rounds: round r decodes the r-th scan of every image
// (a baseline batch is one round), one launch per phase:
//   a. unstuff_kernel     removes the FF00 stuffing and the RSTn markers of every scan (restart segments are byte ranges
//                         the host found)
//   b. Huffman scans (sequential, DC first, AC first with EOB runs), on the scan's own MCU (a non-interleaved scan walks
//      the component's block grid):
//      scan_sync_kernel   self-synchronising Huffman decoding (Weissenberger & Schmidt, ICPP 2018 / HiPC 2021): every
//                         segment is cut into sub_bits-bit subsequences, each decoded speculatively from a guessed state;
//                         sync passes restart a subsequence from its predecessor's exit state until every start state
//                         equals its predecessor's exit state (the state: bit position, block within the MCU, zig-zag index)
//      scan_prefix_kernel prefix sum of the blocks each subsequence completes -> output positions; per-segment checks
//      scan_write_kernel  the final pass: coefficients into their blocks (DC as differences)
//      scan_dc_kernel     DC prediction: a scan per component, reset at every restart
//      dc_refine_kernel   one raw bit per block at a position known from the block's index in its restart segment
//      AC refinement: the bits a block takes depend on which of its coefficients are already nonzero (its history), so
//      no speculative decoder can start mid-segment; the history is fixed before the scan, so the serial part walks
//      registers only:
//      acr_mask_kernel    the history of every block as a 64-bit mask, one thread per block
//      acr_decode_kernel  one warp per restart segment: one lane decodes the symbols against the masks and stores per
//                         block its correction bits and new coefficients; the warp takes long EOB runs 32 blocks a step
//      acr_apply_kernel   corrections and new coefficients into the blocks, one thread per block
//   c. idct_kernel        dequantisation + accurate-integer IDCT (LL&M, 13-bit constants, 2 pass-1 bits), saturated
//   d. colour_kernel      per-component upsampling (libjpeg-turbo's choice of method), the colour conversion of the
//                         frame's colour space (grayscale, YCbCr, RGB, CMYK, YCCK) to BGR, EXIF orientation, uint8 HWC BGR
// oracle/jpeg_numpy.py restates every stage on the CPU, oracle/jpeg_scans_numpy.py the multi-scan entropy decoding,
// oracle/jpeg_colour_numpy.py the frames SMAPB_JPEG_COLOUR adds.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/smap_b200.h"
#include "decode_host.h"
#include "jpeg.h"
#include "orient.h"

namespace smapb {
namespace {

constexpr int SUB_BITS = 512;    // subsequence length of the parallel Huffman decoder
constexpr int WARM_BITS = 1024; // speculative decoding that precedes a subsequence in the first pass
constexpr int PASS_GROUP = 8;    // sync passes launched between two convergence checks on the host
constexpr int GUARD = 8191;      // 16-bit-lane bound of cv2's IDCT (see idct_kernel)
constexpr int MAX_SCAN_BYTES = 1 << 28;  // bit positions are 32-bit

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t h_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct DevHuff {
    uint16_t fast[512];  // next 9 bits -> len << 8 | symbol; 0 = the code is longer (or invalid)
    int32_t maxcode[17];  // largest code of each length 10..16, -1 = none
    int32_t valoff[17];   // vals index of a code of that length = valoff[len] + code
    uint8_t vals[256];
};

constexpr int MAX_COMPS = 4;   // components of a frame
constexpr int MAX_BLOCKS = 10;  // blocks of a frame's MCU (libjpeg's D_MAX_BLOCKS_IN_MCU)

// Colour space of the component planes (libjpeg's jpeg_color_space for the frame)
enum ColourSpace { CS_GRAY = 0, CS_YCC = 1, CS_RGB = 2, CS_CMYK = 3, CS_YCCK = 4 };

struct DevImage {
    int h, w, out_h, out_w, orientation, ncomp, colour, hmax, vmax, mcux, mcuy, nmcu, bpm;
    int blk_comp[MAX_BLOCKS], blk_dx[MAX_BLOCKS], blk_dy[MAX_BLOCKS];
    int comp_h[MAX_COMPS], comp_v[MAX_COMPS];
    int down_w[MAX_COMPS], down_h[MAX_COMPS];  // the component's real (downsampled) size
    int plane_w[MAX_COMPS], plane_h[MAX_COMPS];
    int64_t coef_off, plane_off[MAX_COMPS];
    uint8_t* out;
    int16_t qt[MAX_COMPS][64];  // natural order (values > 32767 are rejected on the host)
};

// A restart segment of a scan; first_mcu / nmcu count the scan's MCUs (single blocks when it is not interleaved).
struct DevSeg {
    int scan, sub0, nsub, first_mcu, nmcu;
    uint32_t bit_begin, bit_end;  // relative to the scan's unstuffed data
};

struct DevSub {
    int scan, seg;
    uint32_t bit_begin, bit_end;
};

enum ScanKind { SCAN_HUFF = 0, SCAN_DC_REFINE = 1, SCAN_AC_REFINE = 2 };

struct DevScan {
    int img, kind, ncomp, bpm, mcux, nmcu, per, inter;
    int tbl_bpm;  // blocks after which the tables repeat: 1 when every block of the MCU uses the same ones
    int ss, se, al;
    int h, v, j0;                 // not interleaved: the component's sampling factors and first block within the frame's MCU
    int blk_comp[MAX_BLOCKS], blk_map[MAX_BLOCKS];  // block of the scan's MCU -> scan component, -> block of the frame's MCU
    int blk_dc[MAX_BLOCKS], blk_ac[MAX_BLOCKS];     // -> its tables (indices into the batch's table array)
    int seg0, nseg, sub0, nsub;
    int acr_off;                  // AC refinement: the scan's first block in the round's masks and records
    int64_t raw_off, raw_len, unst_off;
};

struct SubState {
    unsigned long long start, exit;  // packed decoder states
    int nblk;                        // blocks completed in this subsequence
    int errblk;                      // blocks completed before its first error, INT_MAX = none
};

// packed decoder state: bit position | block within the MCU << 32 | zig-zag index << 40
__host__ __device__ inline unsigned long long pack_state(uint32_t pos, int blk, int zz) {
    return (unsigned long long)pos | ((unsigned long long)blk << 32) | ((unsigned long long)zz << 40);
}

// ---- host parser -----------------------------------------------------------------------------------------------------
struct HuffSpec {
    uint8_t counts[16];
    uint8_t vals[256];
    int nvals = 0;
    bool defined = false;
};

struct Header {
    int h = 0, w = 0, out_h = 0, out_w = 0, orientation = 1, ncomp = 0, hmax = 1, vmax = 1, mcux = 0, mcuy = 0, nmcu = 0;
    int dri = 0, colour = CS_GRAY;
    int comp_h[MAX_COMPS] = {1, 1, 1, 1}, comp_v[MAX_COMPS] = {1, 1, 1, 1};
    uint16_t qt[MAX_COMPS][64];
    HuffSpec dht[2][4];  // the tables defined so far
};

inline int u16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// EXIF orientation from an APP1 payload: 0 = not an EXIF block, 1..8, -1 = an orientation cv2 might read otherwise
int exif_orientation(const uint8_t* s, int64_t len) {
    if (len < 6 || memcmp(s, "Exif\0\0", 6) != 0) return 0;
    return exif_tiff_orientation(s + 6, len - 6);
}

// Validates a Huffman table and fills the device form.  As in libjpeg (jpeg_make_d_derived_tbl), the canonical codes
// must fit their lengths and none may be all ones, so a complete code is refused (cv2 fails on such a file).
bool build_huff(const HuffSpec& s, DevHuff* d) {
    memset(d, 0, sizeof(*d));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; l++) {
        d->valoff[l] = k - code;
        for (int i = 0; i < s.counts[l - 1]; i++) {
            if (code >= (1 << l) - 1) return false;
            if (l <= 9)
                for (int j = 0; j < (1 << (9 - l)); j++) d->fast[(code << (9 - l)) + j] = (uint16_t)((l << 8) | s.vals[k]);
            code++, k++;
        }
        d->maxcode[l] = s.counts[l - 1] ? code - 1 : -1;
        code <<= 1;
    }
    memcpy(d->vals, s.vals, 256);
    return true;
}

constexpr int MAX_SCANS = 64;

struct ScanSpec {
    int ncomp = 0, comp[MAX_COMPS] = {0, 0, 0, 0};  // frame component of each scan component
    int ss = 0, se = 63, ah = 0, al = 0, dri = 0;
    int mcux = 0, nmcu = 0, bpm = 0;     // the scan's MCU grid: the frame's when interleaved, the component's block grid if not
    bool one_table = true;               // every scan component names the same DC and AC tables (libjpeg's CMYK)
    HuffSpec dc[MAX_COMPS], ac[MAX_COMPS];  // the tables in force at this SOS (optimised progressive files redefine them per scan)
    std::vector<int64_t> seg_begin, seg_end;  // raw byte ranges of the restart segments
    std::vector<int64_t> seg_stuffed;         // FF00 pairs inside each segment
};

struct ScanHeader {
    Header f;  // frame geometry, latched quantisers, orientation
    std::vector<ScanSpec> scans;
};

bool huff_ok(const HuffSpec& s) {
    DevHuff d;
    return build_huff(s, &d);
}

// Walks the markers up to EOI.  Without SMAPB_JPEG_SCANS it accepts one interleaved sequential scan (SOF0/SOF1) of every
// component in frame order, followed by EOI.  With it, it also accepts sequential files with several scans (every
// component in exactly one scan) and progressive Huffman files (SOF2) whose progression libjpeg accepts without a warning
// and whose output libjpeg-turbo does not smooth.  Everything else gets a status and goes to cv2.  The two modes report
// some defects at different points (the `!multi` checks), so a file with two defects keeps the status each mode always
// gave it.  SMAPB_JPEG_COLOUR widens the frames either mode accepts: 4 components, 3 components libjpeg treats as RGB,
// and every integral sampling (factors 1..4, at most MAX_BLOCKS blocks per MCU); without it a frame is grayscale or
// YCbCr with luma H, V in {1, 2} and chroma 1x1.
int jpeg_parse(const uint8_t* d, int64_t n, int flags, ScanHeader* M) {
    const bool multi = flags & SMAPB_JPEG_SCANS, colour = flags & SMAPB_JPEG_COLOUR;
    Header* H = &M->f;
    if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) return SMAPB_JPEG_MALFORMED;
    int64_t p = 2;
    const uint8_t* qt[4] = {nullptr, nullptr, nullptr, nullptr};
    int qprec[4] = {0, 0, 0, 0};
    bool sof = false, progressive = false, jfif = false, adobe = false, have_orient = false, qt_used[4] = {false, false, false, false};
    bool latched[MAX_COMPS] = {false, false, false, false};
    int adobe_transform = 0, ids[MAX_COMPS] = {0, 0, 0, 0}, tq[MAX_COMPS] = {0, 0, 0, 0};
    int coef_bits[MAX_COMPS][64];  // libjpeg's progression record: -1 = never coded, else the Al of the last scan that coded it
    int nscanned[MAX_COMPS] = {0, 0, 0, 0};
    memset(coef_bits, 0xFF, sizeof(coef_bits));
    // libjpeg's colour-space rule (default_decompress_parms).  3 components: a JFIF APP0 means YCbCr; else an Adobe APP14
    // means RGB when its transform flag is 0 and YCbCr otherwise; else component ids 'R','G','B' mean RGB, anything else
    // YCbCr.  4 components: an Adobe transform of 2 means YCCK, 0 or no Adobe marker CMYK; libjpeg warns about any other
    // transform and such files are left to cv2.  Without SMAPB_JPEG_COLOUR only grayscale and YCbCr are decoded.
    // -> the colour space, or -1 for a frame left to cv2.
    auto colour_space = [&]() -> int {
        int cs = CS_GRAY;
        if (H->ncomp == 3) {
            if (jfif) cs = CS_YCC;
            else if (adobe) cs = adobe_transform != 0 ? CS_YCC : CS_RGB;
            else cs = ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B' ? CS_RGB : CS_YCC;
        } else if (H->ncomp == 4) {
            cs = !adobe || adobe_transform == 0 ? CS_CMYK : adobe_transform == 2 ? CS_YCCK : -1;
        }
        return colour || cs <= CS_YCC ? cs : -1;
    };
    auto too_large = [&]() { return (int64_t)H->h * H->w > SMAPB_JPEG_MAX_PIXELS; };
    for (;;) {
        if (p + 2 > n || d[p] != 0xFF) return SMAPB_JPEG_MALFORMED;
        while (p + 1 < n && d[p + 1] == 0xFF) p++;
        if (p + 2 > n) return SMAPB_JPEG_MALFORMED;
        const int m = d[p + 1];
        p += 2;
        if (m == 0xD9) {
            if (M->scans.empty()) return SMAPB_JPEG_MALFORMED;
            break;
        }
        if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return SMAPB_JPEG_MALFORMED;
        if (p + 2 > n) return SMAPB_JPEG_MALFORMED;
        int64_t L = u16(d + p);
        if (L < 2 || p + L > n) return SMAPB_JPEG_MALFORMED;
        const uint8_t* s = d + p + 2;
        L -= 2;
        p += L + 2;
        const bool after_scan = !M->scans.empty();
        if (m == 0xDB) {
            for (int64_t i = 0; i < L;) {
                const int pq = s[i] >> 4, t = s[i] & 15;
                if (pq > 1 || t > 3 || i + 1 + 64 * (pq + 1) > L) return SMAPB_JPEG_MALFORMED;
                if (qt_used[t]) return SMAPB_JPEG_UNSUPPORTED;  // a table redefined after a scan latched it
                qt[t] = s + i + 1;
                qprec[t] = pq;
                i += 1 + 64 * (pq + 1);
            }
        } else if (m == 0xC4) {
            for (int64_t i = 0; i < L;) {
                if (i + 17 > L) return SMAPB_JPEG_MALFORMED;
                const int tc = s[i] >> 4, th = s[i] & 15;
                int tot = 0;
                for (int j = 0; j < 16; j++) tot += s[i + 1 + j];
                if (tc > 1 || th > 3 || tot > 256 || i + 17 + tot > L) return SMAPB_JPEG_MALFORMED;
                HuffSpec& hs = H->dht[tc][th];
                memcpy(hs.counts, s + i + 1, 16);
                memset(hs.vals, 0, 256);
                memcpy(hs.vals, s + i + 17, tot);
                hs.nvals = tot;
                hs.defined = true;
                i += 17 + tot;
            }
        } else if (m == 0xDD) {
            if (L != 2) return SMAPB_JPEG_MALFORMED;
            H->dri = u16(s);
        } else if (m == 0xC0 || m == 0xC1 || (m == 0xC2 && multi)) {
            if (sof || L < 6) return SMAPB_JPEG_MALFORMED;
            sof = true;
            progressive = m == 0xC2;
            const int prec = s[0], nf = s[5];
            H->h = u16(s + 1), H->w = u16(s + 3);
            if (L != 6 + 3 * nf) return SMAPB_JPEG_MALFORMED;
            if (prec != 8 || H->h == 0 || H->w == 0 || (nf != 1 && nf != 3 && !(colour && nf == 4)))
                return SMAPB_JPEG_UNSUPPORTED;
            H->ncomp = nf;
            for (int c = 0; c < nf; c++) {
                ids[c] = s[6 + 3 * c];
                H->comp_h[c] = s[7 + 3 * c] >> 4;
                H->comp_v[c] = s[7 + 3 * c] & 15;
                tq[c] = s[8 + 3 * c];
                if (tq[c] > 3) return SMAPB_JPEG_MALFORMED;
                for (int e = 0; e < c; e++)
                    if (ids[e] == ids[c]) return SMAPB_JPEG_MALFORMED;
            }
            if (colour) {
                // libjpeg: factors 1..4 (initial_setup); every ratio to the maxima integral (libjpeg-turbo's upsampler
                // has no fractional one); at most D_MAX_BLOCKS_IN_MCU blocks in an interleaved scan's MCU - frames
                // over it are refused whatever their scans, as the coefficient buffer keeps the frame's MCU
                int hmax = 1, vmax = 1, blocks = 0;
                for (int c = 0; c < nf; c++) {
                    if (H->comp_h[c] < 1 || H->comp_h[c] > 4 || H->comp_v[c] < 1 || H->comp_v[c] > 4)
                        return SMAPB_JPEG_UNSUPPORTED;
                    hmax = std::max(hmax, H->comp_h[c]), vmax = std::max(vmax, H->comp_v[c]);
                    blocks += H->comp_h[c] * H->comp_v[c];
                }
                if (nf > 1) {
                    for (int c = 0; c < nf; c++)
                        if (hmax % H->comp_h[c] || vmax % H->comp_v[c]) return SMAPB_JPEG_UNSUPPORTED;
                    if (blocks > MAX_BLOCKS) return SMAPB_JPEG_UNSUPPORTED;
                }
            }
            if (nf == 1) {
                H->comp_h[0] = H->comp_v[0] = 1;  // one component: one block per MCU whatever its factors say
            } else if (!colour) {
                const bool ok = (H->comp_h[0] == 1 || H->comp_h[0] == 2) && (H->comp_v[0] == 1 || H->comp_v[0] == 2) &&
                                H->comp_h[1] == 1 && H->comp_v[1] == 1 && H->comp_h[2] == 1 && H->comp_v[2] == 1;
                if (!ok) return SMAPB_JPEG_UNSUPPORTED;
            }
            if (multi && too_large()) return SMAPB_JPEG_TOO_LARGE;  // without SMAPB_JPEG_SCANS: at the SOS
            H->hmax = H->vmax = 1;
            for (int c = 0; c < nf; c++) H->hmax = std::max(H->hmax, H->comp_h[c]), H->vmax = std::max(H->vmax, H->comp_v[c]);
            H->mcux = (H->w + 8 * H->hmax - 1) / (8 * H->hmax);
            H->mcuy = (H->h + 8 * H->vmax - 1) / (8 * H->vmax);
            H->nmcu = H->mcux * H->mcuy;
        } else if (m >= 0xC2 && m <= 0xCF) {
            return SMAPB_JPEG_UNSUPPORTED;  // progressive (without SMAPB_JPEG_SCANS), lossless, arithmetic, hierarchical, DAC, JPG
        } else if (m == 0xE0 || m == 0xE1 || m == 0xEE) {
            if (after_scan) return SMAPB_JPEG_UNSUPPORTED;  // colour-space and orientation markers belong before the first scan
            if (m == 0xE0) {
                if (L >= 14 && memcmp(s, "JFIF\0", 5) == 0) jfif = true;
            } else if (m == 0xEE) {
                if (L >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = true, adobe_transform = s[11];
            } else {
                const int o = exif_orientation(s, L);
                if (o < 0) return SMAPB_JPEG_UNSUPPORTED;
                if (o > 0) {
                    if (have_orient) return SMAPB_JPEG_UNSUPPORTED;
                    have_orient = true;
                    H->orientation = o;
                }
            }
        } else if ((m >= 0xE2 && m <= 0xEF) || m == 0xFE) {
        } else if (m == 0xDA) {
            if (!sof) return SMAPB_JPEG_MALFORMED;
            if ((int)M->scans.size() == MAX_SCANS) return SMAPB_JPEG_UNSUPPORTED;
            const int nf = H->ncomp;
            const int ns = L >= 1 ? s[0] : 0;
            if (!multi && (ns != nf || L != 4 + 2 * nf)) return SMAPB_JPEG_UNSUPPORTED;
            if (ns < 1 || ns > nf || L != 4 + 2 * ns) return SMAPB_JPEG_MALFORMED;
            M->scans.emplace_back();
            ScanSpec& S = M->scans.back();
            S.ncomp = ns;
            S.ss = s[1 + 2 * ns], S.se = s[2 + 2 * ns], S.ah = s[3 + 2 * ns] >> 4, S.al = s[3 + 2 * ns] & 15;
            S.dri = H->dri;
            if (multi) {
                for (int k = 0; k < ns; k++) {
                    int c = 0;
                    while (c < nf && ids[c] != s[1 + 2 * k]) c++;
                    if (c == nf || (k > 0 && c <= S.comp[k - 1])) return SMAPB_JPEG_UNSUPPORTED;  // unknown id, or not in frame order
                    S.comp[k] = c;
                }
                if (!progressive) {
                    if (S.ss != 0 || S.se != 63 || S.ah != 0 || S.al != 0) return SMAPB_JPEG_UNSUPPORTED;
                    for (int k = 0; k < ns; k++)
                        if (nscanned[S.comp[k]]++) return SMAPB_JPEG_UNSUPPORTED;
                } else {
                    // libjpeg's checks (start_pass_phuff_decoder): the first group is fatal there, the second a warning
                    // ("bogus progression"); both are left to cv2
                    const bool dc_band = S.ss == 0;
                    if (dc_band ? S.se != 0 : (S.ss > S.se || S.se > 63 || ns != 1)) return SMAPB_JPEG_UNSUPPORTED;
                    if ((S.ah != 0 && S.al != S.ah - 1) || S.al > 13) return SMAPB_JPEG_UNSUPPORTED;
                    for (int k = 0; k < ns; k++) {
                        int* cb = coef_bits[S.comp[k]];
                        if (!dc_band && cb[0] < 0) return SMAPB_JPEG_UNSUPPORTED;
                        for (int i = S.ss; i <= S.se; i++) {
                            if (S.ah != (cb[i] < 0 ? 0 : cb[i])) return SMAPB_JPEG_UNSUPPORTED;
                            cb[i] = S.al;
                        }
                    }
                }
            }
            // without SMAPB_JPEG_SCANS each component is checked in turn (id, tables, quantiser), both tables whatever
            // the band, and the band after them
            const bool dc_first = !multi || (S.ss == 0 && S.ah == 0), uses_ac = !multi || S.se > 0;
            for (int k = 0; k < ns; k++) {
                if (!multi) {
                    if (s[1 + 2 * k] != ids[k]) return SMAPB_JPEG_UNSUPPORTED;
                    S.comp[k] = k;
                }
                const int c = S.comp[k];
                const int td = s[2 + 2 * k] >> 4, ta = s[2 + 2 * k] & 15;
                if (s[2 + 2 * k] != s[2]) S.one_table = false;
                if (!multi && (ta > 3 || !H->dht[1][ta].defined || !qt[tq[c]])) return SMAPB_JPEG_UNSUPPORTED;
                if (dc_first) {
                    if (td > 3 || !H->dht[0][td].defined) return SMAPB_JPEG_UNSUPPORTED;
                    for (int i = 0; i < H->dht[0][td].nvals; i++)
                        if (H->dht[0][td].vals[i] > 15) return SMAPB_JPEG_MALFORMED;
                    S.dc[k] = H->dht[0][td];
                }
                if (uses_ac) {
                    if (ta > 3 || !H->dht[1][ta].defined) return SMAPB_JPEG_UNSUPPORTED;
                    S.ac[k] = H->dht[1][ta];
                }
                if (multi && ((dc_first && !huff_ok(S.dc[k])) || (uses_ac && !huff_ok(S.ac[k])))) return SMAPB_JPEG_MALFORMED;
                if (!latched[c]) {  // libjpeg latches a component's quantiser at its first scan
                    if (!qt[tq[c]]) return SMAPB_JPEG_UNSUPPORTED;
                    for (int i = 0; i < 64; i++) {
                        const int v = qprec[tq[c]] ? u16(qt[tq[c]] + 2 * i) : qt[tq[c]][i];
                        if (v > 32767) return SMAPB_JPEG_UNSUPPORTED;
                        H->qt[c][h_zigzag[i]] = (uint16_t)v;
                    }
                    latched[c] = true;
                    qt_used[tq[c]] = true;
                }
            }
            if (!multi) {
                if (S.ss != 0 || S.se != 63 || S.ah != 0 || S.al != 0) return SMAPB_JPEG_UNSUPPORTED;
                if (colour_space() < 0) return SMAPB_JPEG_UNSUPPORTED;
                if (too_large()) return SMAPB_JPEG_TOO_LARGE;
            }
            if (ns == 1) {  // non-interleaved: the component's own block grid
                const int c = S.comp[0];
                const int cw = (H->w * H->comp_h[c] + H->hmax - 1) / H->hmax, ch = (H->h * H->comp_v[c] + H->vmax - 1) / H->vmax;
                S.mcux = (cw + 7) / 8;
                S.nmcu = S.mcux * ((ch + 7) / 8);
                S.bpm = 1;
            } else {
                S.mcux = H->mcux;
                S.nmcu = H->nmcu;
                S.bpm = 0;
                for (int k = 0; k < ns; k++) S.bpm += H->comp_h[S.comp[k]] * H->comp_v[S.comp[k]];
            }
            const int nseg = S.dri ? (S.nmcu + S.dri - 1) / S.dri : 1;
            // entropy-coded data: FF00 = stuffed FF, FFD0..D7 = restart marker in sequence; any other marker ends the scan,
            // and without SMAPB_JPEG_SCANS it must be EOI
            int64_t start = p, q = p, stuffed = 0;
            for (;;) {
                const uint8_t* f = (const uint8_t*)memchr(d + q, 0xFF, (size_t)(n - q));
                if (!f || f + 1 >= d + n) return SMAPB_JPEG_MALFORMED;
                q = f - d;
                const int mk = d[q + 1];
                if (mk == 0) {
                    stuffed++;
                    q += 2;
                    continue;
                }
                const bool rst = mk >= 0xD0 && mk <= 0xD7;
                if (rst && (!S.dri || mk - 0xD0 != (int)(S.seg_begin.size() % 8) || (int)S.seg_begin.size() + 1 >= nseg))
                    return SMAPB_JPEG_CORRUPT;
                if (!rst && !multi && mk != 0xD9) return SMAPB_JPEG_UNSUPPORTED;
                S.seg_begin.push_back(start);
                S.seg_end.push_back(q);
                S.seg_stuffed.push_back(stuffed);
                if (!rst) break;
                start = q = q + 2;
                stuffed = 0;
            }
            if ((int)S.seg_begin.size() != nseg) return SMAPB_JPEG_CORRUPT;
            if (S.seg_end.back() - S.seg_begin.front() > MAX_SCAN_BYTES) return SMAPB_JPEG_TOO_LARGE;
            p = q;
        } else {
            return SMAPB_JPEG_UNSUPPORTED;
        }
    }
    if (multi) {
        for (int c = 0; c < H->ncomp; c++) {
            if (!progressive) {
                if (nscanned[c] != 1) return SMAPB_JPEG_UNSUPPORTED;
                continue;
            }
            // libjpeg-turbo smooths the output (block smoothing, smoothing_ok) when a component's DC was coded and one of
            // its coefficients 1..9 is not fully refined; those files, and components without DC, are left to cv2
            if (coef_bits[c][0] < 0) return SMAPB_JPEG_UNSUPPORTED;
            for (int i = 1; i <= 9; i++)
                if (coef_bits[c][i] != 0) return SMAPB_JPEG_UNSUPPORTED;
        }
        if (colour_space() < 0) return SMAPB_JPEG_UNSUPPORTED;
    } else {
        // the one scan covers every component and its colour space was checked at its SOS; its tables are checked last
        const ScanSpec& S = M->scans[0];
        for (int k = 0; k < S.ncomp; k++)
            if (!huff_ok(S.dc[k]) || !huff_ok(S.ac[k])) return SMAPB_JPEG_MALFORMED;
    }
    H->colour = colour_space();
    H->out_h = H->orientation >= 5 ? H->w : H->h;
    H->out_w = H->orientation >= 5 ? H->h : H->w;
    return SMAPB_JPEG_OK;
}

// ---- device helpers --------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t peek32(const uint32_t* words, uint32_t pos) {
    const uint32_t w = pos >> 5, sh = pos & 31;
    const uint32_t hi = __byte_perm(words[w], 0, 0x0123), lo = __byte_perm(words[w + 1], 0, 0x0123);
    return __funnelshift_l(lo, hi, sh);
}

// The Huffman code at the top of `bits`: its length (0 = no code of the table) and *sym.  Codes of up to 9 bits come from
// the fast table, longer ones from maxcode.
__device__ __forceinline__ int huff_lookup(const DevHuff& T, uint32_t bits, int* sym) {
    const uint32_t f = T.fast[bits >> 23];
    if (f) {
        *sym = f & 255;
        return f >> 8;
    }
    for (int l = 10; l <= 16; l++) {
        const int code = (int)(bits >> (32 - l));
        if (code <= T.maxcode[l]) {
            *sym = T.vals[(T.valoff[l] + code) & 255];
            return l;
        }
    }
    return 0;
}

// ---- a. unstuffing ---------------------------------------------------------------------------------------------------
// One CTA per scan walks its bytes: a byte is dropped when it follows an FF (the 00 of a stuffed FF, the code byte of
// a restart marker) or when it is an FF that starts a restart marker.  Block-wide prefix sums give the output positions.
__device__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warp_sums[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        const int nw = blockDim.x >> 5;
        int t = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        warp_sums[lane] = t;
    }
    __syncthreads();
    const int before = (wid ? warp_sums[wid - 1] : 0) + x - v;
    *total = warp_sums[(blockDim.x >> 5) - 1];
    __syncthreads();
    return before;
}

constexpr int UNSTUFF_PER_THREAD = 16;

__global__ void __launch_bounds__(1024) unstuff_kernel(const DevScan* __restrict__ scans, const uint8_t* __restrict__ raw,
                                                       uint8_t* __restrict__ unst) {
    const DevScan& I = scans[blockIdx.x];
    const uint8_t* src = raw + I.raw_off;
    uint8_t* dst = unst + I.unst_off;
    const int64_t n = I.raw_len;
    int64_t out = 0;
    for (int64_t base = 0; base < n; base += (int64_t)blockDim.x * UNSTUFF_PER_THREAD) {
        const int64_t i0 = base + (int64_t)threadIdx.x * UNSTUFF_PER_THREAD;
        uint8_t keep[UNSTUFF_PER_THREAD];
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < UNSTUFF_PER_THREAD; k++) {
            const int64_t i = i0 + k;
            bool kp = false;
            if (i < n) {
                const uint8_t b = src[i];
                const bool after_ff = i > 0 && src[i - 1] == 0xFF;
                const bool marker_ff = b == 0xFF && i + 1 < n && src[i + 1] != 0x00;
                kp = !after_ff && !marker_ff;
            }
            keep[k] = kp;
            cnt += kp;
        }
        int total;
        const int at = block_exclusive_scan(cnt, &total);
        int o = 0;
#pragma unroll
        for (int k = 0; k < UNSTUFF_PER_THREAD; k++)
            if (keep[k]) dst[out + at + o++] = src[i0 + k];
        out += total;
    }
    // zero padding behind the data: the bit reader loads whole words past a segment's last bit
    for (int k = threadIdx.x; k < 16; k += blockDim.x) dst[out + k] = 0;
}

// ---- b. Huffman scans and refinement ---------------------------------------------------------------------------------
// Block counts saturate at BLOCK_SAT.  An EOB run adds up to 32767 blocks for 15 bits, so plain
// sums over a scan could pass 2^31; every segment holds far fewer than BLOCK_SAT blocks, so a saturated count is already
// past the segment's end (nothing is written there) and sums of two saturated counts still fit an int.
constexpr int BLOCK_SAT = 1 << 29;

__device__ __forceinline__ int sat_add(int a, int b) { return min(a + b, BLOCK_SAT); }

struct SatAdd {
    __device__ int operator()(int a, int b) const { return sat_add(a, b); }
};
struct IntAdd {
    __device__ int operator()(int a, int b) const { return a + b; }
};

// Block-wide segmented inclusive scan of (head, v), one value per thread in thread order, continued from *carry (the value
// the tiles before this one end with, updated for the next): (h1, v1) + (h2, v2) = (h1 | h2, h2 ? v2 : Add(v1, v2)).
// Every thread of the CTA calls it.
template <class Add>
__device__ int block_segmented_scan(int v, int head, int* carry) {
    __shared__ int s_head[32], s_val[32];
    const Add add;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int x = v, hx = head;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o), hy = __shfl_up_sync(0xffffffffu, hx, o);
        if (lane >= o) {
            if (!hx) x = add(x, y);
            hx |= hy;
        }
    }
    if (lane == 31) s_head[wid] = hx, s_val[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int wx = lane < nw ? s_val[lane] : 0, wh = lane < nw ? s_head[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, wx, o), hy = __shfl_up_sync(0xffffffffu, wh, o);
            if (lane >= o) {
                if (!wh) wx = add(wx, y);
                wh |= hy;
            }
        }
        s_val[lane] = wx, s_head[lane] = wh;
    }
    __syncthreads();
    // prefix from earlier warps of this tile, then the carry of earlier tiles
    if (!hx) {
        if (wid > 0) x = add(x, s_val[wid - 1]);
        if (wid == 0 || !s_head[wid - 1]) x = add(x, *carry);
    }
    const int tile_val = s_val[nw - 1], tile_head = s_head[nw - 1];
    __syncthreads();
    *carry = tile_head ? tile_val : add(*carry, tile_val);
    return x;
}

// The coefficient buffer keeps the single-scan layout (frame MCU by frame MCU, the IDCT reads it as it is); a scan's block
// b (in its own decode order) lands here.
__device__ __forceinline__ int64_t scan_block(const DevScan& S, const DevImage& I, int b) {
    const int m = b / S.bpm, j = b - m * S.bpm;
    if (S.inter) return (int64_t)m * I.bpm + S.blk_map[j];
    const int bx = m % S.mcux, by = m / S.mcux;
    return ((int64_t)(by / S.v) * I.mcux + bx / S.h) * I.bpm + S.j0 + (by % S.v) * S.h + bx % S.h;
}

// Decodes coefficients Ss..Se of each block of one scan from (pos, blk, zz) while pos < stop: DC first / sequential values
// as differences (scan_dc_kernel adds them up), AC values stored << Al.  In progressive AC scans (Ss > 0) an EOBn symbol
// ends a run of 2^n + (n extra bits) blocks; those blocks hold no bits, so the run is counted when its symbol is read and
// the decoder state stays (bit position, block within the MCU, zig-zag index).  Every unit (a Huffman code and its extra
// bits) must end within seg_end.  Errors (a code not in the table, a run past Se, a unit past the segment's end) are
// recorded - `err` = blocks completed before the first one, or -1 - and decoding goes on by a fixed rule (skip one bit; end
// the block; stop), so a speculative decoder that started from a wrong state keeps going until it falls into step with the
// true decoder.  WRITE: coefficients go to the scan's block blk0 + (blocks completed so far); blocks at or beyond `limit`
// are not written.
struct RunResult {
    uint32_t pos;
    int blk, zz, nblk, err;
};

template <bool WRITE>
__device__ RunResult scan_run(const DevScan& S, const DevImage& I, const DevHuff* __restrict__ huffs,
                              const uint32_t* __restrict__ words, uint32_t pos, int blk, int zz, uint32_t stop, uint32_t seg_end,
                              int16_t* __restrict__ coef, int blk0, int limit) {
    int nblk = 0, err = -1;
    const bool eob_runs = S.ss > 0;
    int16_t* b = nullptr;
    int b_at = -1;
    while (pos < stop) {
        const DevHuff& T = huffs[zz == 0 ? S.blk_dc[blk] : S.blk_ac[blk]];
        const uint32_t bits = peek32(words, pos);
        int sym = 0;
        const int len = huff_lookup(T, bits, &sym);
        if (!len) {
            if (err < 0) err = nblk;
            pos++;
            continue;
        }
        const int s = sym & 15, r = sym >> 4;
        const bool eob_n = eob_runs && s == 0 && r < 15;
        const int extra = eob_n ? r : s;
        if ((uint64_t)pos + len + extra > seg_end) {
            if (err < 0) err = nblk;
            pos = seg_end;
            break;
        }
        int v = 0;
        if (extra) {
            v = (int)((bits << len) >> (32 - extra));
            if (!eob_n && v < (1 << (s - 1))) v += 1 - (1 << s);
        }
        if (WRITE && b_at != nblk) {
            b_at = nblk;
            b = blk0 + nblk < limit ? coef + scan_block(S, I, blk0 + nblk) * 64 : nullptr;
        }
        int done = 0;  // blocks this unit completes
        if (zz == 0) {
            if (WRITE && b) b[0] = (int16_t)v;
            zz = 1;
            if (S.se == 0) done = 1;
        } else if (s == 0) {
            if (r == 15) {
                zz += 16;
                if (zz > S.se + 1) {
                    if (err < 0) err = nblk;
                    done = 1;
                } else if (zz == S.se + 1) {
                    done = 1;
                }
            } else {
                done = eob_n ? (1 << r) + v : 1;
            }
        } else {
            zz += r;
            if (zz > S.se) {
                if (err < 0) err = nblk;
                done = 1;
            } else {
                if (WRITE && b) b[c_zigzag[zz]] = (int16_t)((unsigned)v << S.al);
                if (++zz > S.se) done = 1;
            }
        }
        pos += len + extra;
        if (done) {
            zz = S.ss;
            nblk = min(nblk + done, BLOCK_SAT);
            if (++blk == S.tbl_bpm) blk = 0;
        }
    }
    return {pos, blk, zz, nblk, err};
}

// Sync passes over the subsequences [sub_lo, sub_lo + nsub) of one round.
__global__ void __launch_bounds__(256) scan_sync_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                        const DevHuff* __restrict__ huffs, const DevSeg* __restrict__ segs,
                                                        const DevSub* __restrict__ subs, int sub_lo, int nsub,
                                                        const uint8_t* __restrict__ unst, const SubState* __restrict__ prev,
                                                        SubState* __restrict__ cur, int* __restrict__ changed, int pass) {
    if (pass >= 2 && changed[pass - 1] == 0) return;  // converged: the buffer of the first quiet pass is final
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nsub) return;
    const int i = sub_lo + t;
    const DevSub U = subs[i];
    const DevScan& S = scans[U.scan];
    const DevImage& I = imgs[S.img];
    const DevSeg& G = segs[U.seg];
    unsigned long long start;
    if (pass == 0) {
        start = pack_state(U.bit_begin, 0, S.ss);  // a guess, except for the first subsequence of a segment
    } else {
        if (G.sub0 == i) {
            cur[i] = prev[i];
            return;
        }
        start = prev[i - 1].exit;
        if (start == prev[i].start) {
            cur[i] = prev[i];
            return;
        }
    }
    const uint32_t* words = (const uint32_t*)(unst + S.unst_off);
    if (pass == 0 && G.sub0 != i) {
        // warm-up: decode up to WARM_BITS before the subsequence from the guess, so that the state at its first unit
        // boundary has had that long to fall into step with the true decoder
        const uint32_t from = U.bit_begin - min(U.bit_begin - G.bit_begin, (uint32_t)WARM_BITS);
        const RunResult W = scan_run<false>(S, I, huffs, words, from, 0, S.ss, U.bit_begin, G.bit_end, nullptr, 0, 0);
        start = pack_state(W.pos, W.blk, W.zz);
    }
    SubState r;
    r.start = start;
    const RunResult R = scan_run<false>(S, I, huffs, words, (uint32_t)start, (int)(start >> 32) & 255, (int)(start >> 40) & 255,
                                        U.bit_end, G.bit_end, nullptr, 0, 0);
    r.exit = pack_state(R.pos, R.blk, R.zz);
    r.nblk = R.nblk;
    r.errblk = R.err >= 0 ? R.err : 0x7fffffff;
    cur[i] = r;
    changed[pass] = 1;  // benign race: every writer stores 1
}

// One CTA per scan of list[]: base[i] = blocks completed in subsequence i's restart segment up to and including i (a
// segmented, saturating inclusive scan), and the checks that make an image fall back: an error before the segment's last
// block, or fewer blocks than the segment's MCUs hold.
__global__ void __launch_bounds__(1024) scan_prefix_kernel(const DevScan* __restrict__ scans, const int* __restrict__ list,
                                                           const DevSeg* __restrict__ segs, const DevSub* __restrict__ subs,
                                                           const SubState* __restrict__ st, int* __restrict__ base,
                                                           int* __restrict__ status) {
    const DevScan& S = scans[list[blockIdx.x]];
    int carry = 0;
    for (int j0 = 0; j0 < S.nsub; j0 += blockDim.x) {
        const int j = j0 + threadIdx.x;
        int v = 0, head = 0;
        if (j < S.nsub) {
            const int i = S.sub0 + j;
            v = st[i].nblk;
            head = segs[subs[i].seg].sub0 == i;
        }
        const int x = block_segmented_scan<SatAdd>(v, head, &carry);
        if (j < S.nsub) base[S.sub0 + j] = x;
    }
    __syncthreads();
    bool bad = false;
    for (int j = threadIdx.x; j < S.nsub; j += blockDim.x) {
        const int i = S.sub0 + j;
        const SubState s = st[i];
        const DevSeg& G = segs[subs[i].seg];
        if (s.errblk != 0x7fffffff && sat_add(G.sub0 == i ? 0 : base[i - 1], s.errblk) < G.nmcu * S.bpm) bad = true;
        if (i == G.sub0 + G.nsub - 1 && base[i] < G.nmcu * S.bpm) bad = true;  // the segment ends short of its blocks
    }
    if (bad) status[S.img] = SMAPB_JPEG_CORRUPT;
}

__global__ void __launch_bounds__(256) scan_write_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                         const DevHuff* __restrict__ huffs, const DevSeg* __restrict__ segs,
                                                         const DevSub* __restrict__ subs, int sub_lo, int nsub,
                                                         const uint8_t* __restrict__ unst, const SubState* __restrict__ st,
                                                         const int* __restrict__ base, const int* __restrict__ status,
                                                         int16_t* __restrict__ coef) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nsub) return;
    const int i = sub_lo + t;
    const DevSub U = subs[i];
    const DevScan& S = scans[U.scan];
    if (status[S.img] != SMAPB_JPEG_OK) return;
    const DevImage& I = imgs[S.img];
    const DevSeg& G = segs[U.seg];
    const unsigned long long start = st[i].start;
    const int first = G.first_mcu * S.bpm;
    const int local = G.sub0 == i ? 0 : base[i - 1];  // blocks of the segment completed before this subsequence
    const uint32_t* words = (const uint32_t*)(unst + S.unst_off);
    scan_run<true>(S, I, huffs, words, (uint32_t)start, (int)(start >> 32) & 255, (int)(start >> 40) & 255, U.bit_end, G.bit_end,
                   coef + I.coef_off * 64, first + local, first + G.nmcu * S.bpm);
}

// DC prediction of a sequential or DC-first scan: one CTA per (scan, scan component), a segmented scan over that
// component's blocks in decode order, reset at every restart.  The sum runs in int (libjpeg's predictor), the block keeps
// the low 16 bits of (sum << Al).
__global__ void __launch_bounds__(1024) scan_dc_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                       const int* __restrict__ list, const int* __restrict__ status,
                                                       int16_t* __restrict__ coef) {
    const DevScan& S = scans[list[blockIdx.x]];
    const DevImage& I = imgs[S.img];
    const int k = blockIdx.y;
    if (k >= S.ncomp || status[S.img] != SMAPB_JPEG_OK) return;
    int j0 = 0, nc = 0;
    for (int j = 0; j < S.bpm; j++) {
        if (S.blk_comp[j] < k) j0++;
        if (S.blk_comp[j] == k) nc++;
    }
    const int total = S.nmcu * nc;
    int16_t* cf = coef + I.coef_off * 64;
    int carry = 0;
    for (int t0 = 0; t0 < total; t0 += blockDim.x) {
        const int t = t0 + threadIdx.x;
        int v = 0, head = 0;
        int64_t at = 0;
        if (t < total) {
            const int m = t / nc, kk = t % nc;
            at = scan_block(S, I, m * S.bpm + j0 + kk) * 64;
            v = cf[at];
            head = (kk == 0 && m % S.per == 0) ? 1 : 0;
        }
        const int x = block_segmented_scan<IntAdd>(v, head, &carry);
        if (t < total) cf[at] = (int16_t)((unsigned)x << S.al);
    }
}

// DC refinement: one raw bit per block, the n-th bit of its restart segment for the segment's n-th block; sets bit Al.
__global__ void __launch_bounds__(256) dc_refine_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                        const int* __restrict__ list, const DevSeg* __restrict__ segs,
                                                        const uint8_t* __restrict__ unst, int* __restrict__ status,
                                                        int16_t* __restrict__ coef) {
    const DevScan& S = scans[list[blockIdx.y]];
    const DevImage& I = imgs[S.img];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= S.nmcu * S.bpm || status[S.img] != SMAPB_JPEG_OK) return;
    const DevSeg& G = segs[S.seg0 + t / S.bpm / S.per];
    const uint32_t pos = G.bit_begin + (uint32_t)(t - G.first_mcu * S.bpm);
    if (pos >= G.bit_end) {
        status[S.img] = SMAPB_JPEG_CORRUPT;
        return;
    }
    const uint32_t* words = (const uint32_t*)(unst + S.unst_off);
    if (peek32(words, pos) >> 31) {
        int16_t* c = coef + (I.coef_off + scan_block(S, I, t)) * 64;
        c[0] = (int16_t)(c[0] | (1 << S.al));
    }
}

// AC refinement (libjpeg's decode_mcu_AC_refine), in three phases.  The bits a block takes depend only on which of its
// coefficients in [Ss, Se] are nonzero before the scan (its history): one correction bit for every history coefficient the
// decoder passes, and the zero ones count towards a symbol's run.  A coefficient the scan makes nonzero lies behind the
// decoder, so the history stays fixed while the scan is decoded.
//   acr_mask_kernel    one thread per block: its history as a mask, bit k = zig-zag coefficient k, in the scan's order
//   acr_decode_kernel  one warp per restart segment: one lane decodes the symbols against the masks alone, in registers,
//                      and stores per block its correction bits and its new coefficients (AcrRecord); the blocks of an EOB
//                      run past the lane's window of 32 blocks are taken by the whole warp, 32 per step
//   acr_apply_kernel   one thread per block: the corrections and the new +-2^Al coefficients into the coefficient buffer
// A segment's masks and records lie at the scan's acr_off + the segment's first block (these scans are not interleaved).
struct AcrRecord {
    unsigned long long corr;  // bit i: correction bit of the i-th history coefficient (in zig-zag order)
    unsigned long long pos;   // bit k: zig-zag coefficient k becomes +-2^Al
    unsigned long long neg;   // bit k: ... and it is -2^Al
};

constexpr int ACR_WARPS = 4;  // segments per CTA of acr_decode_kernel

__device__ __forceinline__ uint32_t word_be(const uint32_t* words, uint32_t w) { return __byte_perm(words[w], 0, 0x0123); }

// The 64 bits from `pos`, MSB first.
__device__ __forceinline__ unsigned long long peek64(const uint32_t* words, uint32_t pos) {
    const uint32_t w = pos >> 5, sh = pos & 31;
    const uint32_t a = word_be(words, w), b = word_be(words, w + 1), c = word_be(words, w + 2);
    return (unsigned long long)__funnelshift_l(b, a, sh) << 32 | __funnelshift_l(c, b, sh);
}

// The top n bits of v (MSB first) as a word whose bit i is the i-th of them.
__device__ __forceinline__ unsigned long long first_bits_lsb(unsigned long long v, int n) {
    return n ? __brevll(v & ~(~0ull >> n)) : 0ull;
}

// MSB-first bit reader over the unstuffed words: `buf` holds the next `nb` bits (33..64 between calls).
struct BitBuf {
    const uint32_t* words;
    unsigned long long buf;
    int nb;
    uint32_t w, pos;  // next word to load, bit position of buf's first bit
    __device__ __forceinline__ void init(const uint32_t* wd, uint32_t p) {
        words = wd, pos = p, w = p >> 5;
        buf = (unsigned long long)word_be(words, w++) << (32 + (p & 31));
        nb = 32 - (int)(p & 31);
        fill();
    }
    __device__ __forceinline__ void fill() {
        if (nb <= 32) {
            buf |= (unsigned long long)word_be(words, w++) << (32 - nb);
            nb += 32;
        }
    }
    // the next n <= 32 bits, left-aligned
    __device__ __forceinline__ unsigned long long take(int n) {
        const unsigned long long v = buf & ~(~0ull >> n);
        buf <<= n;
        nb -= n, pos += n;
        fill();
        return v;
    }
    // the next n <= 63 bits, left-aligned
    __device__ __forceinline__ unsigned long long take_long(int n) {
        const int a = min(n, 32);
        const unsigned long long hi = take(a);
        return hi | (take(n - a) >> a);
    }
};

__global__ void __launch_bounds__(256) acr_mask_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                       const int* __restrict__ list, const int* __restrict__ status,
                                                       const int16_t* __restrict__ coef, unsigned long long* __restrict__ masks) {
    const DevScan& S = scans[list[blockIdx.y]];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= S.nmcu * S.bpm || status[S.img] != SMAPB_JPEG_OK) return;
    const DevImage& I = imgs[S.img];
    const int4* c = (const int4*)(coef + (I.coef_off + scan_block(S, I, t)) * 64);
    unsigned long long nz = 0;  // natural order
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const int4 v = c[q];
        const int x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; e++)
            nz |= (unsigned long long)((x[e] & 0xFFFF) != 0) << (8 * q + 2 * e) |
                  (unsigned long long)((x[e] >> 16) != 0) << (8 * q + 2 * e + 1);
    }
    unsigned long long m = 0;
    for (int k = S.ss; k <= S.se; k++) m |= (nz >> c_zigzag[k] & 1ull) << k;
    masks[S.acr_off + t] = m;
}

__global__ void __launch_bounds__(32 * ACR_WARPS, 1) acr_decode_kernel(const DevScan* __restrict__ scans,
                                                                    const DevHuff* __restrict__ huffs,
                                                                    const int* __restrict__ list, int n,
                                                                    const DevSeg* __restrict__ segs,
                                                                    const uint8_t* __restrict__ unst, int* __restrict__ status,
                                                                    const unsigned long long* __restrict__ masks,
                                                                    AcrRecord* __restrict__ recs) {
    __shared__ DevHuff s_huff[ACR_WARPS];
    __shared__ unsigned long long s_mask[ACR_WARPS][32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int g = blockIdx.x * ACR_WARPS + wid;
    if (g >= n) return;
    const DevSeg& G = segs[list[g]];
    const DevScan& S = scans[G.scan];
    if (status[S.img] != SMAPB_JPEG_OK) return;
    {
        const uint32_t* src = (const uint32_t*)&huffs[S.blk_ac[0]];
        uint32_t* dst = (uint32_t*)&s_huff[wid];
        for (int i = lane; i < (int)(sizeof(DevHuff) / 4); i += 32) dst[i] = src[i];
    }
    __syncwarp();
    const DevHuff& T = s_huff[wid];
    const uint32_t* words = (const uint32_t*)(unst + S.unst_off);
    const unsigned long long* M = masks + S.acr_off + (int64_t)G.first_mcu * S.bpm;
    AcrRecord* rec = recs + S.acr_off + (int64_t)G.first_mcu * S.bpm;
    const int nblk = G.nmcu * S.bpm;
    const unsigned long long band = (~0ull << S.ss) & (~0ull >> (63 - S.se));  // bits Ss..Se
    const uint32_t end = G.bit_end;
    uint32_t pos = G.bit_begin;
    int run = 0;  // blocks of an open EOB run still to take
    bool bad = false;
    unsigned long long ahead = lane < nblk ? M[lane] : 0ull;  // the next window's masks, one per lane
    for (int q = 0; q < nblk; q += 32) {
        const unsigned long long mine = ahead;
        ahead = q + 32 + lane < nblk ? M[q + 32 + lane] : 0ull;
        const int cnt = min(32, nblk - q);
        int j = 0;
        if (run > 0) {
            // the warp takes the run's blocks of this window: each lane one block, its bits at a warp prefix sum
            j = min(run, cnt);
            const int nb = lane < j ? __popcll(mine) : 0;
            int incl = nb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            if ((uint64_t)pos + total > end) {
                bad = true;
                break;
            }
            if (lane < j) rec[q + lane] = {first_bits_lsb(peek64(words, pos + incl - nb), nb), 0ull, 0ull};
            pos += total;
            run -= j;
        }
        if (j == cnt) continue;
        s_mask[wid][lane] = mine;
        __syncwarp();
        if (lane == 0) {
            BitBuf B;
            B.init(words, pos);
            for (; j < cnt && !bad; j++) {
                const unsigned long long m = s_mask[wid][j];
                if (run > 0) {  // a block of the run: one correction bit per history coefficient
                    const int nc = __popcll(m);
                    if (B.pos + nc > end) {
                        bad = true;
                        break;
                    }
                    rec[q + j] = {first_bits_lsb(B.take_long(nc), nc), 0ull, 0ull};
                    run--;
                    continue;
                }
                // hist / zeros: the history and the zero coefficients of [Ss, Se] the decoder has not passed yet; the
                // correction bits are gathered from bit 63 down and reversed once
                unsigned long long hist = m, zeros = ~m & band, acc = 0, newp = 0, newn = 0;
                int nc = 0;
                for (;;) {
                    int sym = 0;
                    const int len = huff_lookup(T, (uint32_t)(B.buf >> 32), &sym);
                    const int r = sym >> 4, s = sym & 15;
                    // a new coefficient's sign bit follows its code: both are taken at once
                    if (!len || B.pos + len + (s != 0) > end || s > 1) {
                        bad = true;
                        break;
                    }
                    const bool neg = s && (B.buf >> (63 - len) & 1) == 0;
                    B.take(len + s);
                    unsigned long long passed, at = 0;  // the history coefficients the symbol passes, its new coefficient
                    if (!s && r != 15) {  // EOBn: this block's remaining history, then 2^r + extra - 1 more blocks
                        if (B.pos + r > end) {
                            bad = true;
                            break;
                        }
                        run = (1 << r) + (r ? (int)(B.take(r) >> (64 - r)) : 0) - 1;
                        passed = hist;
                    } else {
                        // the (r + 1)-th zero coefficient; a ZRL that finds none passes the rest and ends the block
                        unsigned long long z = zeros;
                        for (int i = 0; i < r && z; i++) z &= z - 1;  // r is 0 for most symbols
                        at = z & (0ull - z);
                        if (s && !at) {
                            bad = true;  // a new coefficient past Se
                            break;
                        }
                        passed = at ? hist & (at - 1) : hist;
                        zeros = z ^ at;
                    }
                    const int nb = __popcll(passed);
                    if (B.pos + nb > end) {
                        bad = true;
                        break;
                    }
                    if (nb) {
                        acc |= (nb <= 32 ? B.take(nb) : B.take_long(nb)) >> nc;
                        nc += nb;
                    }
                    hist ^= passed;
                    if (s) {
                        newp |= at;
                        if (neg) newn |= at;
                    }
                    if (!at || !(zeros | hist)) break;  // EOB, a ZRL that ran out, or Se passed
                }
                const unsigned long long corr = __brevll(acc);
                if (bad) break;
                rec[q + j] = {corr, newp, newn};
            }
            pos = B.pos;
        }
        __syncwarp();
        pos = __shfl_sync(0xffffffffu, pos, 0);
        run = __shfl_sync(0xffffffffu, run, 0);
        if (__shfl_sync(0xffffffffu, (int)bad, 0)) {
            bad = true;
            break;
        }
    }
    if (bad && lane == 0) status[S.img] = SMAPB_JPEG_CORRUPT;
}

__global__ void __launch_bounds__(256) acr_apply_kernel(const DevImage* __restrict__ imgs, const DevScan* __restrict__ scans,
                                                        const int* __restrict__ list, const int* __restrict__ status,
                                                        const unsigned long long* __restrict__ masks,
                                                        const AcrRecord* __restrict__ recs, int16_t* __restrict__ coef) {
    const DevScan& S = scans[list[blockIdx.y]];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= S.nmcu * S.bpm || status[S.img] != SMAPB_JPEG_OK) return;
    const AcrRecord R = recs[S.acr_off + t];
    if (!(R.corr | R.pos)) return;
    const DevImage& I = imgs[S.img];
    int16_t* c = coef + (I.coef_off + scan_block(S, I, t)) * 64;
    const int p1 = 1 << S.al;
    // the i-th correction bit goes with the i-th set bit of the history mask
    unsigned long long m = masks[S.acr_off + t];
    for (unsigned long long corr = R.corr; corr; corr >>= 1, m &= m - 1) {
        if (corr & 1) {
            int16_t* v = c + c_zigzag[__ffsll((long long)m) - 1];
            if ((*v & p1) == 0) *v = (int16_t)(*v >= 0 ? *v + p1 : *v - p1);
        }
    }
    for (unsigned long long p = R.pos; p; p &= p - 1) {
        const int k = __ffsll((long long)p) - 1;
        c[c_zigzag[k]] = (int16_t)(R.neg >> k & 1 ? -p1 : p1);
    }
}

// ---- c. dequantisation + IDCT ----------------------------------------------------------------------------------------
// LL&M 8-point IDCT in 13-bit fixed point (the IJG "accurate integer" method): columns keep 2 extra bits, rows remove
// 13 + 2 + 3 bits; + 128 and saturation to 0..255 (cv2's libjpeg-turbo build saturates, settled on q100 checkerboards).
// cv2's IDCT computes in 16-bit lanes; where a dequantised coefficient or a pass-1 output leaves +-GUARD one of them could
// overflow, and the image is left to cv2 (never happens with encoder-written quantisers).
struct Idct8 {
    int o[8];
};

__device__ __forceinline__ Idct8 idct8(int x0, int x1, int x2, int x3, int x4, int x5, int x6, int x7, int shift) {
    int z1 = (x2 + x6) * 4433;
    const int t2 = z1 - x6 * 15137, t3 = z1 + x2 * 6270;
    const int t0 = (x0 + x4) * 8192, t1 = (x0 - x4) * 8192;
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int a0 = x7, a1 = x5, a2 = x3, a3 = x1;
    z1 = a0 + a3;
    int z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
    const int z5 = (z3 + z4) * 9633;
    a0 *= 2446, a1 *= 16819, a2 *= 25172, a3 *= 12299;
    z1 *= -7373, z2 *= -20995, z3 = z3 * -16069 + z5, z4 = z4 * -3196 + z5;
    a0 += z1 + z3, a1 += z2 + z4, a2 += z2 + z3, a3 += z1 + z4;
    const int r = 1 << (shift - 1);
    Idct8 R;
    R.o[0] = (t10 + a3 + r) >> shift, R.o[7] = (t10 - a3 + r) >> shift;
    R.o[1] = (t11 + a2 + r) >> shift, R.o[6] = (t11 - a2 + r) >> shift;
    R.o[2] = (t12 + a1 + r) >> shift, R.o[5] = (t12 - a1 + r) >> shift;
    R.o[3] = (t13 + a0 + r) >> shift, R.o[4] = (t13 - a0 + r) >> shift;
    return R;
}

__global__ void __launch_bounds__(128) idct_kernel(const DevImage* __restrict__ imgs, const int16_t* __restrict__ coef,
                                                   uint8_t* __restrict__ planes, int* __restrict__ status) {
    const DevImage& I = imgs[blockIdx.y];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= I.nmcu * I.bpm || status[blockIdx.y] != SMAPB_JPEG_OK) return;
    const int m = g / I.bpm, j = g % I.bpm, c = I.blk_comp[j];
    const int bx = (m % I.mcux) * I.comp_h[c] + I.blk_dx[j], by = (m / I.mcux) * I.comp_v[c] + I.blk_dy[j];
    const int4* src = (const int4*)(coef + (I.coef_off + g) * 64);
    int x[64];
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int4 q = src[r];
        const int w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            x[r * 8 + 2 * k] = (int)(int16_t)(w4[k] & 0xFFFF) * I.qt[c][r * 8 + 2 * k];
            x[r * 8 + 2 * k + 1] = (int)(int16_t)((unsigned)w4[k] >> 16) * I.qt[c][r * 8 + 2 * k + 1];
        }
    }
    bool over = false;
#pragma unroll
    for (int k = 0; k < 64; k++) over |= x[k] > GUARD || x[k] < -GUARD;
#pragma unroll
    for (int col = 0; col < 8; col++) {
        const Idct8 R = idct8(x[col], x[8 + col], x[16 + col], x[24 + col], x[32 + col], x[40 + col], x[48 + col], x[56 + col], 11);
#pragma unroll
        for (int r = 0; r < 8; r++) {
            x[r * 8 + col] = R.o[r];
            over |= R.o[r] > GUARD || R.o[r] < -GUARD;
        }
    }
    if (over) {
        status[blockIdx.y] = SMAPB_JPEG_UNSUPPORTED;
        return;
    }
    uint8_t* dst = planes + I.plane_off[c] + (int64_t)by * 8 * I.plane_w[c] + bx * 8;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const Idct8 R = idct8(x[r * 8], x[r * 8 + 1], x[r * 8 + 2], x[r * 8 + 3], x[r * 8 + 4], x[r * 8 + 5], x[r * 8 + 6],
                              x[r * 8 + 7], 18);
        uint32_t lo = 0, hi = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            lo |= (uint32_t)min(max(R.o[k] + 128, 0), 255) << (8 * k);
            hi |= (uint32_t)min(max(R.o[k + 4] + 128, 0), 255) << (8 * k);
        }
        *(uint2*)(dst + (int64_t)r * I.plane_w[c]) = make_uint2(lo, hi);
    }
}

// ---- d. upsampling, colour, orientation ------------------------------------------------------------------------------
__device__ __forceinline__ int px(const uint8_t* p, int pw, int y, int x) { return p[(int64_t)y * pw + x]; }

// Component c at the frame's pixel (y, x), upsampled by the method libjpeg-turbo 3.x picks for it (jinit_upsampler), from
// its factors (h, v) and the frame's maxima: equal factors as is; twice as wide (same height) fancy h2v1, twice as tall
// (same width) fancy h1v2, both fancy h2v2 - the h2 filters only when the component is more than 2 samples wide, else
// replication; any other integral ratio replication (int_upsample).  Fancy filters clamp at the component's real size.
__device__ int sample_at(const DevImage& I, const uint8_t* __restrict__ planes, int c, int y, int x) {
    const uint8_t* C = planes + I.plane_off[c];
    const int pw = I.plane_w[c], h = I.comp_h[c], v = I.comp_v[c], cw = I.down_w[c], ch = I.down_h[c];
    if (h == I.hmax && v == I.vmax) return px(C, pw, y, x);
    const bool h2 = 2 * h == I.hmax && cw > 2, v2 = 2 * v == I.vmax;
    if (h2 && v == I.vmax) {  // h2v1
        const int i = x >> 1, n = (x & 1) ? min(i + 1, cw - 1) : max(i - 1, 0);
        return (3 * px(C, pw, y, i) + px(C, pw, y, n) + ((x & 1) ? 2 : 1)) >> 2;
    }
    if (v2 && h == I.hmax) {  // h1v2
        const int r0 = y >> 1, r1 = (y & 1) ? min(r0 + 1, ch - 1) : max(r0 - 1, 0);
        return (3 * px(C, pw, r0, x) + px(C, pw, r1, x) + ((y & 1) ? 2 : 1)) >> 2;
    }
    if (h2 && v2) {  // h2v2: column sums of the nearer and the further row
        const int i = x >> 1, n = (x & 1) ? min(i + 1, cw - 1) : max(i - 1, 0);
        const int r0 = y >> 1, r1 = (y & 1) ? min(r0 + 1, ch - 1) : max(r0 - 1, 0);
        const int s0 = 3 * px(C, pw, r0, i) + px(C, pw, r1, i), s1 = 3 * px(C, pw, r0, n) + px(C, pw, r1, n);
        return (3 * s0 + s1 + ((x & 1) ? 7 : 8)) >> 4;
    }
    return px(C, pw, y / (I.vmax / v), x / (I.hmax / h));
}

// JFIF YCbCr -> RGB with 16-bit fixed-point constants round(k * 2^16), rounded by adding 2^15, saturated
__device__ __forceinline__ void ycc_rgb(int Y, int cb, int cr, int* r, int* g, int* b) {
    cb -= 128, cr -= 128;
    *r = min(max(Y + ((91881 * cr + 32768) >> 16), 0), 255);
    *g = min(max(Y + ((-46802 * cr - 22554 * cb + 32768) >> 16), 0), 255);
    *b = min(max(Y + ((116130 * cb + 32768) >> 16), 0), 255);
}

// cv2's CMYK -> BGR (icvCvt_CMYK2BGR_8u_C4C3R) of one ink
__device__ __forceinline__ int ink(int x, int k) { return k - (((255 - x) * k) >> 8); }

// libjpeg's conversion to what cv2 asks for (BGR from 1 or 3 components, CMYK from 4), then cv2's CMYK -> BGR:
//   grayscale  replicated          YCbCr  the tables above          RGB  reordered
//   CMYK       as stored           YCCK   C, M, Y = 255 - the R, G, B of (Y, Cb, Cr), K as stored
__global__ void __launch_bounds__(256) colour_kernel(const DevImage* __restrict__ imgs, const uint8_t* __restrict__ planes,
                                                     const int* __restrict__ status) {
    const DevImage& I = imgs[blockIdx.y];
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)I.h * I.w || status[blockIdx.y] != SMAPB_JPEG_OK) return;
    const int y = (int)(t / I.w), x = (int)(t % I.w);
    const int s0 = sample_at(I, planes, 0, y, x);
    int b = s0, g = s0, r = s0;
    if (I.ncomp > 1) {
        const int s1 = sample_at(I, planes, 1, y, x), s2 = sample_at(I, planes, 2, y, x);
        if (I.colour == CS_RGB) {
            r = s0, g = s1, b = s2;
        } else if (I.colour == CS_CMYK) {
            const int k = sample_at(I, planes, 3, y, x);
            r = ink(s0, k), g = ink(s1, k), b = ink(s2, k);
        } else {
            ycc_rgb(s0, s1, s2, &r, &g, &b);
            if (I.colour == CS_YCCK) {
                const int k = sample_at(I, planes, 3, y, x);
                r = ink(255 - r, k), g = ink(255 - g, k), b = ink(255 - b, k);
            }
        }
    }
    int oy, ox;
    orient_store_pos(I.orientation, I.h, I.w, y, x, &oy, &ox);
    uint8_t* o = I.out + ((int64_t)oy * I.out_w + ox) * 3;
    o[0] = (uint8_t)b, o[1] = (uint8_t)g, o[2] = (uint8_t)r;
}

}  // namespace

// staging: descriptors and scan bytes; small: status[m] then changed[passes]
struct JpegWorkspace {
    PinnedBuffer<uint8_t> host;
    DeviceBuffer<uint8_t> dev_in;
    DeviceBuffer<int> small;
    PinnedBuffer<int> small_host;
    DeviceBuffer<uint8_t> unst;
    DeviceBuffer<SubState> st[2];
    DeviceBuffer<int> base;
    DeviceBuffer<int16_t> coef;
    DeviceBuffer<unsigned long long> acr_mask;  // AC refinement: history masks and records of a round's blocks
    DeviceBuffer<AcrRecord> acr_rec;
    DeviceBuffer<uint8_t> planes;
    int sub_bits = SUB_BITS;  // subsequence length of the Huffman passes (SMAPB_JPEG_SUB_BITS)
};

JpegWorkspace* jpeg_workspace_create() {
    JpegWorkspace* ws = new JpegWorkspace();
    if (const char* e = getenv("SMAPB_JPEG_SUB_BITS")) {
        const int v = atoi(e);
        if (v >= 32 && v % 32 == 0) ws->sub_bits = v;
    }
    return ws;
}

void jpeg_workspace_destroy(JpegWorkspace* ws) { delete ws; }

namespace {
// What one round (the r-th scan of every image that has one) launches: subsequences [sub_lo, sub_lo + nsub) of its
// Huffman scans, and ranges of the batch's index list (scans, and segments for AC refinement).  AC refinement scans
// take acr_total blocks of the masks and records, the largest acr_blocks.
struct Round {
    int sub_lo = 0, nsub = 0, max_nsub_seg = 1;
    int huff_off = 0, nhuff = 0, dc_off = 0, ndc = 0, dcr_off = 0, ndcr = 0, dcr_blocks = 0, acr_off = 0, nacr = 0;
    int acrs_off = 0, nacrs = 0, acr_blocks = 0, acr_total = 0;
};
}  // namespace

int jpeg_decode(JpegWorkspace* ws, int n, const uint8_t* const* jpeg, const int64_t* nbytes, uint8_t* const* bgr, int flags,
                int* status, cudaStream_t st, int64_t* launches, std::string* err) {
    // host: parse, then lay out descriptors and scan bytes
    std::vector<ScanHeader> H;
    std::vector<int> idx;  // images that go to the device
    const auto walk = [flags](const uint8_t* d, int64_t nb, ScanHeader* M) { return jpeg_parse(d, nb, flags, M); };
    const int m = decode_preamble("smapb_decode_jpeg_ex", n, jpeg, nbytes, bgr, status, st, walk, &H, &idx, err);
    if (m <= 0) return m;
    std::vector<DevImage> imgs(m);
    std::vector<DevScan> scans;
    std::vector<DevHuff> huffs;
    std::vector<DevSeg> segs;
    std::vector<DevSub> subs;
    std::vector<int> lists;
    int64_t raw_total = 0, unst_total = 0, coef_blocks = 0, plane_total = 0;
    int max_blocks = 0, nrounds = 0;
    int64_t max_px = 0;
    for (int k = 0; k < m; k++) {
        const Header& h = H[idx[k]].f;
        DevImage& I = imgs[k];
        memset(&I, 0, sizeof(I));
        I.h = h.h, I.w = h.w, I.out_h = h.out_h, I.out_w = h.out_w, I.orientation = h.orientation, I.ncomp = h.ncomp;
        I.colour = h.colour;
        I.hmax = h.hmax, I.vmax = h.vmax, I.mcux = h.mcux, I.mcuy = h.mcuy, I.nmcu = h.nmcu;
        I.out = bgr[idx[k]];
        int j = 0;
        for (int c = 0; c < h.ncomp; c++) {
            for (int v = 0; v < h.comp_v[c]; v++)
                for (int u = 0; u < h.comp_h[c]; u++) I.blk_comp[j] = c, I.blk_dx[j] = u, I.blk_dy[j] = v, j++;
            I.comp_h[c] = h.comp_h[c], I.comp_v[c] = h.comp_v[c];
            I.down_w[c] = (h.w * h.comp_h[c] + h.hmax - 1) / h.hmax;
            I.down_h[c] = (h.h * h.comp_v[c] + h.vmax - 1) / h.vmax;
            I.plane_w[c] = h.mcux * h.comp_h[c] * 8;
            I.plane_h[c] = h.mcuy * h.comp_v[c] * 8;
            I.plane_off[c] = plane_total;
            plane_total += align_up((size_t)I.plane_w[c] * I.plane_h[c], 256);
            for (int q = 0; q < 64; q++) I.qt[c][q] = (int16_t)h.qt[c][q];
        }
        I.bpm = j;
        I.coef_off = coef_blocks;
        coef_blocks += (int64_t)h.nmcu * I.bpm;
        max_blocks = std::max(max_blocks, h.nmcu * I.bpm);
        max_px = std::max(max_px, (int64_t)h.h * h.w);
        nrounds = std::max(nrounds, (int)H[idx[k]].scans.size());
    }
    // scans round by round, so that every round's subsequences are contiguous
    std::vector<Round> rounds(nrounds);
    std::vector<int> huff_l, dc_l, dcr_l, acr_l, acrs_l;
    int acr_max = 0;  // blocks of the masks and records: the most any round needs
    for (int r = 0; r < nrounds; r++) {
        Round& R = rounds[r];
        R.sub_lo = (int)subs.size();
        huff_l.clear(), dc_l.clear(), dcr_l.clear(), acr_l.clear(), acrs_l.clear();
        for (int k = 0; k < m; k++) {
            const ScanHeader& M = H[idx[k]];
            if ((int)M.scans.size() <= r) continue;
            const ScanSpec& P = M.scans[r];
            const Header& h = M.f;
            const int si = (int)scans.size();
            DevScan D;
            memset(&D, 0, sizeof(D));
            D.img = k;
            D.kind = P.ah == 0 ? SCAN_HUFF : P.ss == 0 ? SCAN_DC_REFINE : SCAN_AC_REFINE;
            D.ncomp = P.ncomp, D.bpm = P.bpm, D.mcux = P.mcux, D.nmcu = P.nmcu, D.per = P.dri ? P.dri : P.nmcu;
            D.inter = P.ncomp > 1;
            D.ss = P.ss, D.se = P.se, D.al = P.al;
            int j = 0;
            for (int q = 0; q < P.ncomp; q++) {
                const int c = P.comp[q];
                int dc = 0, ac = 0;
                if (D.kind == SCAN_HUFF && P.ss == 0) {
                    dc = (int)huffs.size();
                    huffs.emplace_back();
                    build_huff(P.dc[q], &huffs.back());
                }
                if (D.kind != SCAN_DC_REFINE && P.se > 0) {
                    ac = (int)huffs.size();
                    huffs.emplace_back();
                    build_huff(P.ac[q], &huffs.back());
                }
                int j0c = 0;
                for (int e = 0; e < c; e++) j0c += h.comp_h[e] * h.comp_v[e];
                for (int v = 0; v < h.comp_v[c]; v++)
                    for (int u = 0; u < h.comp_h[c]; u++)
                        D.blk_comp[j] = q, D.blk_map[j] = j0c + v * h.comp_h[c] + u, D.blk_dc[j] = dc, D.blk_ac[j] = ac, j++;
                D.h = h.comp_h[c], D.v = h.comp_v[c], D.j0 = j0c;  // used when the scan has one component
            }
            if (!D.inter) D.bpm = 1;
            // the decoder state keeps the block within the MCU only to pick its tables; when they are all the same the
            // bits cannot tell the blocks apart, and a speculative decoder would never fall into step with that index
            D.tbl_bpm = P.one_table ? 1 : D.bpm;
            D.raw_off = raw_total;
            D.raw_len = P.seg_end.back() - P.seg_begin.front();
            raw_total += align_up(D.raw_len, 16);
            D.unst_off = unst_total;
            D.seg0 = (int)segs.size();
            D.sub0 = (int)subs.size();
            D.nseg = (int)P.seg_begin.size();
            uint32_t bit = 0;
            for (int s = 0; s < D.nseg; s++) {
                const int64_t len = P.seg_end[s] - P.seg_begin[s] - P.seg_stuffed[s];
                DevSeg G;
                G.scan = si;
                G.first_mcu = s * D.per;
                G.nmcu = std::min(D.per, D.nmcu - G.first_mcu);
                G.bit_begin = bit;
                G.bit_end = bit + (uint32_t)(len * 8);
                G.sub0 = (int)subs.size();
                G.nsub = 0;
                if (D.kind == SCAN_HUFF) {
                    G.nsub = std::max(1, (int)((len * 8 + ws->sub_bits - 1) / ws->sub_bits));
                    for (int u = 0; u < G.nsub; u++) {
                        DevSub U;
                        U.scan = si;
                        U.seg = (int)segs.size();
                        U.bit_begin = std::min(G.bit_end, G.bit_begin + (uint32_t)u * ws->sub_bits);
                        U.bit_end = u == G.nsub - 1 ? G.bit_end : G.bit_begin + (uint32_t)(u + 1) * ws->sub_bits;
                        subs.push_back(U);
                    }
                    R.max_nsub_seg = std::max(R.max_nsub_seg, G.nsub);
                } else if (D.kind == SCAN_AC_REFINE) {
                    acr_l.push_back((int)segs.size());
                }
                segs.push_back(G);
                bit = G.bit_end;
            }
            D.nsub = (int)subs.size() - D.sub0;
            unst_total += align_up(bit / 8 + 16, 16);
            if (D.kind == SCAN_HUFF) {
                huff_l.push_back(si);
                if (P.ss == 0) dc_l.push_back(si);
            } else if (D.kind == SCAN_DC_REFINE) {
                dcr_l.push_back(si);
                R.dcr_blocks = std::max(R.dcr_blocks, D.nmcu * D.bpm);
            } else {
                acrs_l.push_back(si);
                D.acr_off = R.acr_total;
                R.acr_total += D.nmcu * D.bpm;
                R.acr_blocks = std::max(R.acr_blocks, D.nmcu * D.bpm);
            }
            scans.push_back(D);
        }
        R.nsub = (int)subs.size() - R.sub_lo;
        auto put = [&](const std::vector<int>& v, int* off, int* cnt) {
            *off = (int)lists.size(), *cnt = (int)v.size();
            lists.insert(lists.end(), v.begin(), v.end());
        };
        put(huff_l, &R.huff_off, &R.nhuff);
        put(dc_l, &R.dc_off, &R.ndc);
        put(dcr_l, &R.dcr_off, &R.ndcr);
        put(acr_l, &R.acr_off, &R.nacr);
        put(acrs_l, &R.acrs_off, &R.nacrs);
        acr_max = std::max(acr_max, R.acr_total);
    }
    const int nscan = (int)scans.size();
    int max_passes = 1;
    for (const Round& R : rounds) max_passes = std::max(max_passes, R.max_nsub_seg + 1);
    // staging layout: images | scans | tables | segments | subsequences | lists | scan bytes
    const size_t o_img = 0, o_scan = align_up(o_img + sizeof(DevImage) * m, 256),
                 o_huff = align_up(o_scan + sizeof(DevScan) * nscan, 256),
                 o_seg = align_up(o_huff + sizeof(DevHuff) * huffs.size(), 256),
                 o_sub = align_up(o_seg + sizeof(DevSeg) * segs.size(), 256),
                 o_list = align_up(o_sub + sizeof(DevSub) * subs.size(), 256),
                 o_raw = align_up(o_list + sizeof(int) * lists.size(), 256), total = o_raw + raw_total;
    DECODE_CK(ws->host.grow(total));
    DECODE_CK(cudaStreamSynchronize(st));  // the staging area and the workspace may still be in use by the previous call
    memcpy(ws->host + o_img, imgs.data(), sizeof(DevImage) * m);
    memcpy(ws->host + o_scan, scans.data(), sizeof(DevScan) * nscan);
    memcpy(ws->host + o_huff, huffs.data(), sizeof(DevHuff) * huffs.size());
    memcpy(ws->host + o_seg, segs.data(), sizeof(DevSeg) * segs.size());
    memcpy(ws->host + o_sub, subs.data(), sizeof(DevSub) * subs.size());
    memcpy(ws->host + o_list, lists.data(), sizeof(int) * lists.size());
    {
        int si = 0;
        for (int r = 0; r < nrounds; r++)
            for (int k = 0; k < m; k++) {
                const ScanHeader& M = H[idx[k]];
                if ((int)M.scans.size() <= r) continue;
                const ScanSpec& P = M.scans[r];
                memcpy(ws->host + o_raw + scans[si].raw_off, jpeg[idx[k]] + P.seg_begin.front(), scans[si].raw_len);
                si++;
            }
    }
    const size_t nsub = std::max<size_t>(1, subs.size());
    DECODE_CK(ws->dev_in.grow(total));
    DECODE_CK(ws->unst.grow((size_t)unst_total));
    DECODE_CK(ws->st[0].grow(nsub));
    DECODE_CK(ws->st[1].grow(nsub));
    DECODE_CK(ws->base.grow(nsub));
    DECODE_CK(ws->coef.grow((size_t)coef_blocks * 64));
    DECODE_CK(ws->planes.grow((size_t)plane_total));
    if (acr_max) {
        DECODE_CK(ws->acr_mask.grow((size_t)acr_max));
        DECODE_CK(ws->acr_rec.grow((size_t)acr_max));
    }
    DECODE_CK(ws->small.grow((size_t)m + max_passes + PASS_GROUP));
    DECODE_CK(ws->small_host.grow((size_t)m + PASS_GROUP));
    const DevImage* d_img = (const DevImage*)(ws->dev_in + o_img);
    const DevScan* d_scan = (const DevScan*)(ws->dev_in + o_scan);
    const DevHuff* d_huff = (const DevHuff*)(ws->dev_in + o_huff);
    const DevSeg* d_seg = (const DevSeg*)(ws->dev_in + o_seg);
    const DevSub* d_sub = (const DevSub*)(ws->dev_in + o_sub);
    const int* d_list = (const int*)(ws->dev_in + o_list);
    const uint8_t* d_raw = ws->dev_in + o_raw;
    int* d_status = ws->small;
    int* d_changed = ws->small + m;
    for (int k = 0; k < m; k++) ws->small_host[k] = status[idx[k]];
    DECODE_CK(cudaMemcpyAsync(ws->dev_in, ws->host, total, cudaMemcpyHostToDevice, st));
    DECODE_CK(cudaMemcpyAsync(d_status, ws->small_host, sizeof(int) * m, cudaMemcpyHostToDevice, st));
    DECODE_CK(cudaMemsetAsync(ws->coef, 0, (size_t)coef_blocks * 64 * sizeof(int16_t), st));
    unstuff_kernel<<<nscan, 1024, 0, st>>>(d_scan, d_raw, ws->unst);
    DECODE_CK(cudaGetLastError());
    ++*launches;
    for (const Round& R : rounds) {
        if (R.nsub) {
            DECODE_CK(cudaMemsetAsync(d_changed, 0, sizeof(int) * (max_passes + PASS_GROUP), st));
            const int round_passes = R.max_nsub_seg + 1;
            const int sgrid = (R.nsub + 255) / 256;
            int pass = 0, final_pass = -1;
            while (final_pass < 0) {
                const int stop = std::min(pass + PASS_GROUP, round_passes + 1);
                const int first = pass;
                for (; pass < stop; pass++) {
                    scan_sync_kernel<<<sgrid, 256, 0, st>>>(d_img, d_scan, d_huff, d_seg, d_sub, R.sub_lo, R.nsub, ws->unst,
                                                            ws->st[(pass + 1) & 1], ws->st[pass & 1], d_changed, pass);
                    DECODE_CK(cudaGetLastError());
                    ++*launches;
                }
                DECODE_CK(cudaMemcpyAsync(ws->small_host, d_changed + first, sizeof(int) * (stop - first), cudaMemcpyDeviceToHost,
                                          st));
                DECODE_CK(cudaStreamSynchronize(st));
                for (int p = first; p < stop; p++)
                    if (p > 0 && ws->small_host[p - first] == 0) {
                        final_pass = p;
                        break;
                    }
                if (final_pass < 0 && pass > round_passes) {
                    *err = "smapb_decode_jpeg_ex: Huffman sync passes did not converge";
                    return -11;
                }
            }
            const SubState* fin = ws->st[final_pass & 1];
            scan_prefix_kernel<<<R.nhuff, 1024, 0, st>>>(d_scan, d_list + R.huff_off, d_seg, d_sub, fin, ws->base, d_status);
            scan_write_kernel<<<sgrid, 256, 0, st>>>(d_img, d_scan, d_huff, d_seg, d_sub, R.sub_lo, R.nsub, ws->unst, fin, ws->base,
                                                     d_status, ws->coef);
            DECODE_CK(cudaGetLastError());
            *launches += 2;
        }
        if (R.ndc) {
            scan_dc_kernel<<<dim3(R.ndc, MAX_COMPS), 1024, 0, st>>>(d_img, d_scan, d_list + R.dc_off, d_status, ws->coef);
            DECODE_CK(cudaGetLastError());
            ++*launches;
        }
        if (R.ndcr) {
            dc_refine_kernel<<<dim3((R.dcr_blocks + 255) / 256, R.ndcr), 256, 0, st>>>(d_img, d_scan, d_list + R.dcr_off, d_seg,
                                                                                       ws->unst, d_status, ws->coef);
            DECODE_CK(cudaGetLastError());
            ++*launches;
        }
        if (R.nacr) {
            const dim3 grid((R.acr_blocks + 255) / 256, R.nacrs);
            acr_mask_kernel<<<grid, 256, 0, st>>>(d_img, d_scan, d_list + R.acrs_off, d_status, ws->coef, ws->acr_mask);
            acr_decode_kernel<<<(R.nacr + ACR_WARPS - 1) / ACR_WARPS, 32 * ACR_WARPS, 0, st>>>(
                d_scan, d_huff, d_list + R.acr_off, R.nacr, d_seg, ws->unst, d_status, ws->acr_mask, ws->acr_rec);
            acr_apply_kernel<<<grid, 256, 0, st>>>(d_img, d_scan, d_list + R.acrs_off, d_status, ws->acr_mask, ws->acr_rec,
                                                   ws->coef);
            DECODE_CK(cudaGetLastError());
            *launches += 3;
        }
    }
    idct_kernel<<<dim3((max_blocks + 127) / 128, m), 128, 0, st>>>(d_img, ws->coef, ws->planes, d_status);
    colour_kernel<<<dim3((unsigned)((max_px + 255) / 256), m), 256, 0, st>>>(d_img, ws->planes, d_status);
    DECODE_CK(cudaGetLastError());
    *launches += 2;
    DECODE_CK(cudaMemcpyAsync(ws->small_host, d_status, sizeof(int) * m, cudaMemcpyDeviceToHost, st));
    DECODE_CK(cudaStreamSynchronize(st));
    for (int k = 0; k < m; k++)
        if (status[idx[k]] == SMAPB_JPEG_OK) status[idx[k]] = ws->small_host[k];
    return 0;
}

}  // namespace smapb

extern "C" {
#pragma GCC visibility push(default)
int smapb_jpeg_info_ex(const uint8_t* data, int64_t nbytes, int flags, int* h, int* w, int* orientation, int* status) {
    if (!status || (flags & ~(SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR))) return -1;
    smapb::ScanHeader M;
    return smapb::report_info(smapb::jpeg_parse(data, nbytes, flags, &M), M.f, status, h, w, orientation);
}

int smapb_jpeg_info(const uint8_t* data, int64_t nbytes, int* h, int* w, int* orientation, int* status) {
    return smapb_jpeg_info_ex(data, nbytes, 0, h, w, orientation, status);
}
#pragma GCC visibility pop
}
