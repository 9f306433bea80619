// EXIF orientation, shared by the JPEG and PNG decoders: the TIFF-block parser on the host and the store position on the
// device.  A JPEG carries the TIFF block in APP1 behind "Exif\0\0", a PNG in its eXIf chunk as it is.
#pragma once
#include <stdint.h>
#include <string.h>

namespace smapb {

// Orientation tag of a TIFF block: 1..8, 1 when the block has no such tag, -1 = a block or a value cv2 might read otherwise
inline int exif_tiff_orientation(const uint8_t* t, int64_t n) {
    if (n < 8) return -1;
    bool le;
    if (memcmp(t, "II*\0", 4) == 0) le = true;
    else if (memcmp(t, "MM\0*", 4) == 0) le = false;
    else return -1;
    auto rd = [&](int64_t i, int k, bool* ok) -> uint32_t {
        if (i < 0 || i + k > n) {
            *ok = false;
            return 0;
        }
        uint32_t v = 0;
        for (int j = 0; j < k; j++) v |= (uint32_t)t[i + j] << (8 * (le ? j : k - 1 - j));
        return v;
    };
    bool ok = true;
    const int64_t ifd = rd(4, 4, &ok);
    const int cnt = (int)rd(ifd, 2, &ok);
    if (!ok) return -1;
    for (int e = 0; e < cnt; e++) {
        const int64_t p = ifd + 2 + 12 * (int64_t)e;
        const uint32_t tag = rd(p, 2, &ok);
        if (!ok) return -1;
        if (tag == 0x0112) {
            const uint32_t typ = rd(p + 2, 2, &ok), c = rd(p + 4, 4, &ok), v = rd(p + 8, 2, &ok);
            if (!ok || typ != 3 || c != 1 || v < 1 || v > 8) return -1;
            return (int)v;
        }
    }
    return 1;
}

#ifdef __CUDACC__
// Where pixel (y, x) of an h x w image lands in the oriented output, as cv2 applies the EXIF orientation (2 flip x,
// 3 rotate 180, 4 flip y, 5 transpose, 6 rotate 90 cw, 7 transverse, 8 rotate 90 ccw)
__device__ __forceinline__ void orient_store_pos(int orientation, int h, int w, int y, int x, int* oy, int* ox) {
    *oy = y, *ox = x;
    switch (orientation) {
        case 2: *ox = w - 1 - x; break;
        case 3: *oy = h - 1 - y, *ox = w - 1 - x; break;
        case 4: *oy = h - 1 - y; break;
        case 5: *oy = x, *ox = y; break;
        case 6: *oy = x, *ox = h - 1 - y; break;
        case 7: *oy = w - 1 - x, *ox = h - 1 - y; break;
        case 8: *oy = w - 1 - x, *ox = y; break;
        default: break;
    }
}
#endif

}  // namespace smapb
