"""CPU restatement of smap_b200/csrc/png.cu: the chunk walk, the CRCs, the inflate (Python's zlib), the unfilter, the pixel
conversions and the EXIF orientation of cv2.imdecode(buf, IMREAD_COLOR).

decode(buf) -> (status, image): status is one of the SMAPB_JPEG_* values the GPU decoder reports, image the uint8 BGR
[H, W, 3] array when status is OK, else None.  parse(buf) -> (status, header) is the host walk alone (smapb_png_info)."""
import struct
import zlib

import numpy as np

OK, UNSUPPORTED, MALFORMED, CORRUPT, TOO_LARGE = 0, 1, 2, 3, 4
MAX_PIXELS = 1 << 26
MAX_STREAM_BYTES = 1 << 28
SIG = b"\x89PNG\r\n\x1a\n"
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# Adam7: first row, first column, row step, column step of each pass
ADAM7 = [(0, 0, 8, 8), (0, 4, 8, 8), (4, 0, 8, 4), (0, 2, 4, 4), (2, 0, 4, 2), (0, 1, 2, 2), (1, 0, 2, 1)]


def tiff_orientation(t):
    """Orientation tag of a TIFF block: 1..8, 1 without the tag, -1 = unreadable (smapb::exif_tiff_orientation)."""
    n = len(t)
    if n < 8:
        return -1
    if t[:4] == b"II*\0":
        e = "<"
    elif t[:4] == b"MM\0*":
        e = ">"
    else:
        return -1

    def rd(i, k):
        if i < 0 or i + k > n:
            raise IndexError
        return struct.unpack(e + ("H" if k == 2 else "I"), t[i:i + k])[0]

    try:
        ifd = rd(4, 4)
        cnt = rd(ifd, 2)
        for k in range(cnt):
            p = ifd + 2 + 12 * k
            if rd(p, 2) == 0x0112:
                typ, c, v = rd(p + 2, 2), rd(p + 4, 4), rd(p + 8, 2)
                return v if typ == 3 and c == 1 and 1 <= v <= 8 else -1
    except IndexError:
        return -1
    return 1


def parse(b):
    """-> (status, header dict or None)."""
    if len(b) < 8 or b[:8] != SIG:
        return MALFORMED, None
    H = dict(orientation=1, pal=bytes(768), idat=[], plte=False)
    p, n = 8, len(b)
    ihdr = exif = iend = idat_done = False
    while p < n:
        if n - p < 12:
            return MALFORMED, None
        ln = struct.unpack(">I", b[p:p + 4])[0]
        t = b[p + 4:p + 8]
        if ln > 0x7fffffff or ln > n - p - 12:
            return MALFORMED, None
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in t):
            return MALFORMED, None
        s = b[p + 8:p + 8 + ln]
        crc = struct.unpack(">I", b[p + 8 + ln:p + 12 + ln])[0]
        if not ihdr and t != b"IHDR":
            return MALFORMED, None
        if t != b"IDAT" and zlib.crc32(t + s) != crc:
            return CORRUPT, None
        if H["idat"] and t != b"IDAT":
            idat_done = True
        if t == b"IHDR":
            if ihdr or ln != 13:
                return MALFORMED, None
            ihdr = True
            w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", s)
            if not (w and h and w <= 0x7fffffff and h <= 0x7fffffff and depth in DEPTHS.get(ctype, ()) and comp == 0 and
                    filt == 0 and inter <= 1):
                return MALFORMED, None
            if w * h > MAX_PIXELS:
                return TOO_LARGE, None
            H.update(w=w, h=h, depth=depth, ctype=ctype, interlace=inter)
        elif t == b"PLTE":
            if H["plte"] or H["idat"] or H["ctype"] in (0, 4):
                return UNSUPPORTED, None
            if ln == 0 or ln % 3 or ln > 768:
                return MALFORMED, None
            H["plte"] = True
            if H["ctype"] == 3:
                if ln // 3 > 1 << H["depth"]:
                    return UNSUPPORTED, None
                H["pal"] = s + bytes(768 - ln)
        elif t == b"IDAT":
            if idat_done:
                return UNSUPPORTED, None
            if H["ctype"] == 3 and not H["plte"]:
                return MALFORMED, None
            H["idat"].append((s, crc))
        elif t == b"IEND":
            if ln:
                return MALFORMED, None
            iend = True
            break
        elif t == b"eXIf":
            if exif:
                return UNSUPPORTED, None
            exif = True
            o = tiff_orientation(s)
            if o < 0:
                return UNSUPPORTED, None
            H["orientation"] = o
        elif t in (b"acTL", b"fcTL", b"fdAT"):
            return UNSUPPORTED, None
        elif not t[0] & 0x20:
            return UNSUPPORTED, None
        p += 12 + ln
    if not (ihdr and iend and H["idat"]):
        return MALFORMED, None
    z = b"".join(s for s, _ in H["idat"])
    if len(z) > MAX_STREAM_BYTES:
        return TOO_LARGE, None
    if len(z) < 2:
        return CORRUPT, None
    if z[0] & 15 != 8 or z[0] >> 4 > 7 or ((z[0] << 8) | z[1]) % 31:
        return CORRUPT, None
    if z[1] & 0x20:
        return UNSUPPORTED, None
    H["z"] = z
    H["out_shape"] = (H["w"], H["h"]) if H["orientation"] >= 5 else (H["h"], H["w"])
    return OK, H


def passes(H):
    """[(width, height)] of the scanline groups: the image, or the 7 Adam7 passes (empty ones as (0, 0))."""
    if not H["interlace"]:
        return [(H["w"], H["h"])]
    out = []
    for ys, xs, dy, dx in ADAM7:
        pw, ph = (H["w"] - xs + dx - 1) // dx, (H["h"] - ys + dy - 1) // dy
        out.append((pw, ph) if pw > 0 and ph > 0 else (0, 0))
    return out


def row_bytes(H, pw):
    return (pw * CHANNELS[H["ctype"]] * H["depth"] + 7) // 8


def unfilter(rows, rb, bpp, data):
    """data: ph scanlines of 1 + rb bytes -> uint8 [ph, rb]; None for a filter type > 4."""
    out = np.zeros((rows, rb), np.int32)
    d = np.frombuffer(data, np.uint8).reshape(rows, rb + 1).astype(np.int32)
    prev = np.zeros(rb, np.int32)
    for r in range(rows):
        f, x = d[r, 0], d[r, 1:]
        if f > 4:
            return None
        if f == 0:
            cur = x.copy()
        elif f == 2:
            cur = (x + prev) & 255
        else:
            cur = np.zeros(rb, np.int32)
            for i in range(rb):
                a = cur[i - bpp] if i >= bpp else 0
                b = prev[i]
                c = prev[i - bpp] if i >= bpp else 0
                if f == 1:
                    v = a
                elif f == 3:
                    v = (a + b) >> 1
                else:
                    pp = a + b - c
                    pa, pb, pc = abs(pp - a), abs(pp - b), abs(pp - c)
                    v = a if pa <= pb and pa <= pc else b if pb <= pc else c
                cur[i] = (x[i] + v) & 255
        out[r] = cur
        prev = cur
    return out.astype(np.uint8)


def to_bgr(H, rows, pw):
    """Unfiltered scanlines of one pass -> uint8 BGR [ph, pw, 3] (cv2's IMREAD_COLOR conversions)."""
    depth, ctype, ch = H["depth"], H["ctype"], CHANNELS[H["ctype"]]
    ph = rows.shape[0]
    if depth < 8:
        bits = np.unpackbits(rows, axis=1)[:, :pw * depth].reshape(ph, pw, depth)
        v = (bits * (1 << np.arange(depth - 1, -1, -1))).sum(-1)
        if ctype == 3:
            pal = np.frombuffer(H["pal"], np.uint8).reshape(256, 3)
            rgb = pal[v]
        else:
            g = (v * 255 // ((1 << depth) - 1)).astype(np.uint8)
            rgb = np.stack([g, g, g], -1)
    else:
        s = rows[:, :pw * ch * depth // 8].reshape(ph, pw, ch, depth // 8)[..., 0]  # 16-bit: the high byte
        if ctype == 3:
            rgb = np.frombuffer(H["pal"], np.uint8).reshape(256, 3)[s[..., 0]]
        elif ctype in (0, 4):
            rgb = np.repeat(s[..., :1], 3, -1)
        else:
            rgb = s[..., :3]
    return np.ascontiguousarray(rgb[..., ::-1]).astype(np.uint8)


def orient(img, o):
    """EXIF orientation as cv2 applies it."""
    return {1: img, 2: img[:, ::-1], 3: img[::-1, ::-1], 4: img[::-1], 5: img.transpose(1, 0, 2),
            6: img.transpose(1, 0, 2)[:, ::-1], 7: img.transpose(1, 0, 2)[::-1, ::-1], 8: img.transpose(1, 0, 2)[::-1]}[o]


def inflate(H):
    """-> (status, scanline bytes).  zlib decides validity; the stream must end exactly after its Adler-32 and yield
    exactly the bytes the scanlines need."""
    need = sum(ph * (1 + row_bytes(H, pw)) for pw, ph in passes(H) if pw)
    for s, crc in H["idat"]:
        if zlib.crc32(b"IDAT" + s) != crc:
            return CORRUPT, None
    d = zlib.decompressobj()
    try:
        out = d.decompress(H["z"])
    except zlib.error:
        return CORRUPT, None
    if not d.eof or len(out) < need:
        return CORRUPT, None
    if len(out) > need or d.unused_data:
        return UNSUPPORTED, None
    return OK, out


def decode(b):
    st, H = parse(b)
    if st != OK:
        return st, None
    st, raw = inflate(H)
    if st != OK:
        return st, None
    img = np.zeros((H["h"], H["w"], 3), np.uint8)
    off = 0
    for p, (pw, ph) in enumerate(passes(H)):
        if not pw:
            continue
        rb = row_bytes(H, pw)
        rows = unfilter(ph, rb, max(1, CHANNELS[H["ctype"]] * H["depth"] // 8), raw[off:off + ph * (rb + 1)])
        if rows is None:
            return CORRUPT, None
        off += ph * (rb + 1)
        bgr = to_bgr(H, rows, pw)
        if H["interlace"]:
            ys, xs, dy, dx = ADAM7[p]
            img[ys::dy, xs::dx] = bgr
        else:
            img = bgr
    return OK, np.ascontiguousarray(orient(img, H["orientation"]))
