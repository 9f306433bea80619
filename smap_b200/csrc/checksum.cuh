// CRC-32 (PNG chunks) and Adler-32 (zlib streams) pieces shared by the PNG decoder (png.cu) and encoder (png_enc.cu).
// A CRC over a byte range is computed in slices from a zero register; slice k is shifted over the bytes after it by a
// multiplication with x^(8 n) mod P, and the slices and the shifted initial register are XORed (zlib's crc32_combine).
#pragma once
#include <stdint.h>

namespace smapb {

constexpr uint32_t ADLER_MOD = 65521;

// the byte-wise CRC-32 table entry of i (reflected polynomial 0xEDB88320)
__host__ __device__ __forceinline__ uint32_t crc_table_entry(uint32_t i) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    return c;
}

inline uint32_t crc32_host(const uint8_t* p, int64_t n) {
    static uint32_t T[256];
    static bool init = false;
    if (!init) {
        for (uint32_t i = 0; i < 256; i++) T[i] = crc_table_entry(i);
        init = true;
    }
    uint32_t c = 0xFFFFFFFFu;
    for (int64_t i = 0; i < n; i++) c = T[(c ^ p[i]) & 255] ^ (c >> 8);
    return ~c;
}

__device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {  // a * b modulo the CRC-32 polynomial (reflected)
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

// x^(8 n) mod P from the table x2n[k] = x^(2^k) mod P
__device__ __forceinline__ uint32_t x8nmodp(const uint32_t* x2n, uint64_t n) {
    uint32_t p = 1u << 31;  // x^0
    int k = 3;
    while (n) {
        if (n & 1) p = multmodp(x2n[k & 31], p);
        n >>= 1;
        k++;
    }
    return p;
}

// Fills the shared tables T[256] (byte-wise CRC) and x2n[32] with the CTA; ends with __syncthreads.
__device__ __forceinline__ void crc_tables(uint32_t* T, uint32_t* x2n) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) T[i] = crc_table_entry(i);
    if (threadIdx.x == 0) {
        uint32_t p = 1u << 30;  // x^1
        x2n[0] = p;
        for (int k = 1; k < 32; k++) x2n[k] = p = multmodp(p, p);
    }
    __syncthreads();
}

// One thread's share of the CRC-32 of L bytes read by get(j): its slice, shifted over the bytes after it.  XOR the shares
// of every thread of the CTA (blockDim.x of them) with the shifted initial register (crc_finish) to get the CRC.
template <typename Get>
__device__ __forceinline__ uint32_t crc_slice(const uint32_t* T, const uint32_t* x2n, uint64_t L, Get get) {
    const uint64_t S = (L + blockDim.x - 1) / blockDim.x;
    const uint64_t a = min(L, (uint64_t)threadIdx.x * S), b = min(L, a + S);
    uint32_t r = 0;
    for (uint64_t j = a; j < b; j++) r = T[(r ^ get(j)) & 255] ^ (r >> 8);
    if (a < b && b < L) r = multmodp(x8nmodp(x2n, L - b), r);
    return r;
}

// The CRC from the XOR of every thread's crc_slice over L bytes.
__device__ __forceinline__ uint32_t crc_finish(const uint32_t* x2n, uint64_t L, uint32_t shares) {
    return ~(multmodp(x8nmodp(x2n, L), 0xFFFFFFFFu) ^ shares);
}

}  // namespace smapb
