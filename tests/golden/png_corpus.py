"""Seeded PNG corpus for the GPU decoder's tests (tests/test_png_cpu.py, tests/test_png_gpu.py), written at test time by a
small PNG writer (struct + zlib), cv2.imencode and Pillow: every bit depth / colour type pair with and without Adam7,
every filter type on every row and mixed filters, zlib levels, strategies, memLevels, windows and flushes, split IDATs,
eXIf orientations and ancillary chunks, sizes from 1x1 up; damaged() adds files cv2 refuses or the decoder leaves to it."""
import io
import struct
import zlib

import numpy as np

from jpeg_corpus import content, exif_block

PAIRS = [(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16), (6, 8),
         (6, 16)]  # (colour type, bit depth)
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
ADAM7 = [(0, 0, 8, 8), (0, 4, 8, 8), (4, 0, 8, 4), (0, 2, 4, 4), (2, 0, 4, 2), (0, 1, 2, 2), (1, 0, 2, 1)]


def chunk(t, d):
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)


def samples(ctype, depth, h, w, rng, kind="smooth"):
    """Sample array [h, w, channels] (uint16 for 16-bit) with smooth or noisy content."""
    ch, top = CHANNELS[ctype], (1 << depth) - 1
    if kind == "noise" or depth < 8:
        return rng.integers(0, top + 1, (h, w, ch)).astype(np.uint16 if depth == 16 else np.uint8)
    base = content("smooth", h, w, rng).astype(np.int64)
    s = np.concatenate([base, 255 - base[..., :1]], -1)[..., :ch] if ch != 2 else base[..., :3:2]
    if depth == 16:
        return (s * 257 + rng.integers(0, 256, s.shape)).astype(np.uint16)
    return s.astype(np.uint8)


def pack_rows(s, depth):
    """[h, w, ch] samples -> list of packed scanline bytes (no filter byte)."""
    h, w, ch = s.shape
    if depth == 16:
        return [s[r].astype(">u2").tobytes() for r in range(h)]
    if depth == 8:
        return [s[r].tobytes() for r in range(h)]
    rows = []
    for r in range(h):
        bits = ((s[r, :, 0][:, None] >> np.arange(depth - 1, -1, -1)) & 1).astype(np.uint8).ravel()
        rows.append(np.packbits(bits).tobytes())
    return rows


def filter_rows(rows, bpp, filters):
    """Applies the filter filters(r) to each row -> filtered bytes with filter bytes."""
    out, prev = bytearray(), None
    for r, row in enumerate(rows):
        x = np.frombuffer(row, np.uint8).astype(np.int32)
        p = np.zeros_like(x) if prev is None else prev
        a = np.concatenate([np.zeros(bpp, np.int32), x[:-bpp]]) if len(x) > bpp else np.zeros_like(x)
        c = np.concatenate([np.zeros(bpp, np.int32), p[:-bpp]]) if len(x) > bpp else np.zeros_like(x)
        f = filters(r)
        if f == 0:
            y = x
        elif f == 1:
            y = x - a
        elif f == 2:
            y = x - p
        elif f == 3:
            y = x - ((a + p) >> 1)
        else:
            pp = a + p - c
            pa, pb, pc = abs(pp - a), abs(pp - p), abs(pp - c)
            y = x - np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, p, c))
        out += bytes([f]) + (y & 255).astype(np.uint8).tobytes()
        prev = x
    return bytes(out)


def scanlines(s, ctype, depth, interlace, filters):
    bpp = max(1, CHANNELS[ctype] * depth // 8)
    if not interlace:
        return filter_rows(pack_rows(s, depth), bpp, filters)
    out = b""
    for ys, xs, dy, dx in ADAM7:
        sub = s[ys::dy, xs::dx]
        if sub.size:
            out += filter_rows(pack_rows(sub, depth), bpp, filters)
    return out


def compress(raw, level=6, wbits=15, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY, flush=None, pieces=1):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits, mem, strategy)
    out, step = b"", max(1, -(-len(raw) // pieces))
    for i in range(0, len(raw), step):
        out += c.compress(raw[i:i + step])
        if flush is not None and i + step < len(raw):
            out += c.flush(flush)
    return out + c.flush()


def write_png(s, ctype, depth, interlace=0, filters=lambda r: r % 5, z=None, zopts=None, split=None, pre=b"", post=b"",
              palette=None, empty_after=0):
    """A PNG of the samples: IHDR, `pre` chunks, PLTE, IDAT(s) cut into pieces of the sizes split(i) gives (0 = an empty
    IDAT), `empty_after` empty IDATs, `post`, IEND."""
    h, w = s.shape[:2]
    if z is None:
        z = compress(scanlines(s, ctype, depth, interlace, filters), **(zopts or {}))
    b = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace)) + pre
    if ctype == 3:
        b += chunk(b"PLTE", palette if palette is not None else bytes(range(256)) * 3 if depth == 8 else
                   bytes((i * 37 + k * 91) % 256 for i in range(1 << depth) for k in range(3)))
    if split is None:
        b += chunk(b"IDAT", z)
    else:
        i, k = 0, 0
        while i < len(z):
            n = split(k)
            b += chunk(b"IDAT", z[i:i + n])
            i, k = i + n, k + 1
    b += chunk(b"IDAT", b"") * empty_after
    return b + post + chunk(b"IEND", b"")


def cv2_png(img, level=None):
    import cv2

    p = [] if level is None else [cv2.IMWRITE_PNG_COMPRESSION, level]
    ok, b = cv2.imencode(".png", img, p)
    assert ok
    return b.tobytes()


def pil_png(img_bgr, **kw):
    from PIL import Image

    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img_bgr[:, :, ::-1])).save(bio, "PNG", **kw)
    return bio.getvalue()


def exif_chunk(o, big_endian=False):
    return chunk(b"eXIf", exif_block(o, big_endian)[6:])


def corpus(seed=0, large=False):
    """[(name, bytes)] of files the GPU decoder must decode to cv2's bytes."""
    rng = np.random.default_rng(seed)
    out = []
    for ctype, depth in PAIRS:
        for inter in (0, 1):
            for h, w in ((1, 1), (3, 5), (13, 11), (37, 61)):
                s = samples(ctype, depth, h, w, rng, "noise" if w < 20 else "smooth")
                out.append(("t%d_d%d_i%d_%dx%d" % (ctype, depth, inter, h, w), write_png(s, ctype, depth, inter)))
    s = samples(2, 8, 40, 33, rng)
    for f in range(5):
        out.append(("filter%d_every_row" % f, write_png(s, 2, 8, 0, filters=lambda r, f=f: f)))
        out.append(("filter%d_every_row_gray2" % f, write_png(samples(0, 2, 9, 23, rng), 0, 2, 0, filters=lambda r, f=f: f)))
    out.append(("mixed_filters_adam7", write_png(s, 2, 8, 1, filters=lambda r: (r * 7 + 3) % 5)))
    img = content("smooth", 96, 128, rng)
    raw_s = samples(2, 8, 96, 128, rng)
    for lvl in range(10):
        out.append(("zlib_level%d" % lvl, write_png(raw_s, 2, 8, zopts=dict(level=lvl))))
        out.append(("cv2_level%d" % lvl, cv2_png(img, lvl)))
    for name, st in (("rle", zlib.Z_RLE), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("fixed", zlib.Z_FIXED),
                     ("filtered", zlib.Z_FILTERED)):
        out.append(("strategy_" + name, write_png(raw_s, 2, 8, zopts=dict(strategy=st))))
    for mem in (1, 9):
        out.append(("memlevel%d" % mem, write_png(raw_s, 2, 8, zopts=dict(mem=mem))))
    for wb in (9, 10, 12, 14):
        out.append(("window%d" % wb, write_png(raw_s, 2, 8, zopts=dict(wbits=wb))))
    for name, fl in (("sync", zlib.Z_SYNC_FLUSH), ("partial", zlib.Z_PARTIAL_FLUSH), ("full", zlib.Z_FULL_FLUSH)):
        out.append(("flush_" + name, write_png(raw_s, 2, 8, zopts=dict(flush=fl, pieces=7))))
    out.append(("idat_1byte", write_png(samples(2, 8, 20, 17, rng), 2, 8, split=lambda k: 1)))
    out.append(("idat_odd", write_png(raw_s, 2, 8, split=lambda k: 1 + (k * 997) % 4093)))
    for o in range(1, 9):
        out.append(("exif%d" % o, write_png(samples(2, 8, 7, 12, rng), 2, 8, pre=exif_chunk(o, o % 2 == 0))))
    out.append(("exif6_after_idat", write_png(samples(2, 8, 7, 12, rng), 2, 8, post=exif_chunk(6))))
    anc = (chunk(b"gAMA", struct.pack(">I", 100000)) + chunk(b"sBIT", bytes([5, 6, 5])) + chunk(b"tEXt", b"k\x00v") +
           chunk(b"pHYs", bytes(9)) + chunk(b"bKGD", bytes(6)))
    out.append(("ancillary", write_png(samples(2, 8, 9, 10, rng), 2, 8, pre=anc, post=chunk(b"tIME", bytes(7)))))
    out.append(("trns_rgb", write_png(samples(2, 8, 5, 6, rng), 2, 8, pre=chunk(b"tRNS", bytes(6)))))
    pal_trns = write_png(samples(3, 8, 5, 6, rng), 3, 8)
    i = pal_trns.find(b"IDAT") - 4
    out.append(("trns_palette", pal_trns[:i] + chunk(b"tRNS", bytes(range(10))) + pal_trns[i:]))
    out.append(("palette_short", write_png(samples(3, 8, 6, 9, rng), 3, 8, palette=bytes(range(30)))))
    out.append(("pil", pil_png(content("smooth", 50, 70, rng))))
    out.append(("pil_optimize", pil_png(content("noise", 30, 40, rng), optimize=True)))
    out.append(("cv2_gray16", cv2_png((content("smooth", 20, 30, rng)[..., 0].astype(np.uint16) * 257))))
    if large:
        for h, w in ((1080, 1920), (3024, 4032)):
            im = content("smooth", h, w, rng)
            out.append(("cv2_%dx%d" % (w, h), cv2_png(im)))
            out.append(("zlib6_%dx%d" % (w, h), write_png(im[..., ::-1], 2, 8, filters=lambda r: 4, zopts=dict(level=6))))
        out.append(("adam7_rgba16_640x480", write_png(samples(6, 16, 480, 640, rng), 6, 16, 1)))
    return out


def large_frames(seed=1, n=8, sizes=((1080, 1920), (3024, 4032))):
    """[(name, bytes)] of the benchmark's frames: cv2.imencode defaults and zlib level 6 (Paeth rows, as PIL writes)."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        for k in range(n):
            im = content("smooth", h, w, rng)
            if k % 2 == 0:
                out.append(("cv2_%dx%d_%d" % (w, h, k), cv2_png(im)))
            else:
                out.append(("zlib6_%dx%d_%d" % (w, h, k), write_png(im[..., ::-1], 2, 8, filters=lambda r: 4)))
    return out


def damaged(seed=2):
    """[(name, bytes)]: cuts in every chunk and inside the stream, flipped CRCs, a bad Adler-32, too little and too much
    data, bad zlib headers, APNG, unknown critical chunks."""
    rng = np.random.default_rng(seed)
    s = samples(2, 8, 24, 31, rng)
    raw = scanlines(s, 2, 8, 0, lambda r: r % 5)
    good = write_png(s, 2, 8, z=zlib.compress(raw), pre=chunk(b"tEXt", b"a\x00b") + exif_chunk(3))
    out = []
    p = 8
    while p < len(good):
        ln = struct.unpack(">I", good[p:p + 4])[0]
        t = good[p + 4:p + 8].decode()
        for cut in (p + 2, p + 6, p + 8 + ln // 2, p + 10 + ln):
            out.append(("cut_%s_%d" % (t, cut - p), good[:cut]))
        flip = bytearray(good)
        flip[p + 8 + ln] ^= 0x10
        out.append(("crc_%s" % t, bytes(flip)))
        p += 12 + ln
    z = bytearray(zlib.compress(raw))
    z[-1] ^= 1
    out.append(("bad_adler", write_png(s, 2, 8, z=bytes(z))))
    out.append(("too_little", write_png(s, 2, 8, z=zlib.compress(raw[:-40]))))
    out.append(("too_much", write_png(s, 2, 8, z=zlib.compress(raw + bytes(50)))))
    out.append(("bytes_after_adler", write_png(s, 2, 8, z=zlib.compress(raw) + b"\x00\x00")))
    zc = zlib.compress(raw)
    for k in range(0, len(zc) - 4, max(1, len(zc) // 12)):
        out.append(("stream_cut_%d" % k, write_png(s, 2, 8, z=zc[:k])))
        fl = bytearray(zc)
        fl[k] ^= 0x5a
        out.append(("stream_flip_%d" % k, write_png(s, 2, 8, z=bytes(fl))))
    for name, hdr in (("cinfo8", 0x88), ("cm7", 0x77)):
        b1 = (31 - (hdr * 256) % 31) % 31
        out.append(("zhdr_" + name, write_png(s, 2, 8, z=bytes([hdr, b1]) + zc[2:])))
    out.append(("zhdr_check", write_png(s, 2, 8, z=bytes([zc[0], zc[1] ^ 1]) + zc[2:])))
    out.append(("zhdr_fdict", write_png(s, 2, 8, z=bytes([0x78, 0xbb]) + b"\x00\x00\x00\x01" + zc[2:])))
    out.append(("apng", write_png(s, 2, 8, z=zc, pre=chunk(b"acTL", struct.pack(">II", 1, 0)))))
    out.append(("unknown_critical", write_png(s, 2, 8, z=zc, pre=chunk(b"ABCD", b"x"))))
    out.append(("bad_filter", write_png(s, 2, 8, z=zlib.compress(b"\x07" + raw[1:]))))
    out.append(("plte_in_gray", write_png(samples(0, 8, 3, 4, rng), 0, 8, pre=chunk(b"PLTE", bytes(6)))))
    out.append(("not_png", b"GIF89a" + bytes(40)))
    out.append(("empty", b""))
    return out
