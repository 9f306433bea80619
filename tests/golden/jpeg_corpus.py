"""Seeded JPEG corpus for the GPU decoder's tests (tests/test_jpeg_cpu.py, tests/test_jpeg_gpu.py), written by cv2 and
Pillow at test time: sizes, qualities, samplings, grayscale, restart intervals, optimised tables, 16-bit DQT, EXIF
orientations, flat / noise / checkerboard / smooth content; plus files the decoder must leave to cv2."""
import io

import numpy as np

SAMPLINGS = {"420": 0x221111, "422": 0x211111, "440": 0x121111, "444": 0x111111}  # cv2.IMWRITE_JPEG_SAMPLING_FACTOR_*
SMALL = [(1, 1), (5, 7), (8, 8), (9, 17), (37, 61)]  # (h, w)


def content(kind, h, w, rng):
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "check":
        yy, xx = np.mgrid[:h, :w]
        c = (((yy + xx) % 2) * 255).astype(np.uint8)
        return np.stack([c, 255 - c, c], 2)
    # smooth: gradients with mild noise (large frames at a moderate entropy)
    yy, xx = np.mgrid[:h, :w]
    base = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 127 // max(h + w - 2, 1)], 2)
    return np.clip(base + rng.integers(-6, 7, (h, w, 3)), 0, 255).astype(np.uint8)


def cv2_jpeg(img, q=90, samp="420", rst=0, optimize=False):
    import cv2

    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[samp]]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    ok, b = cv2.imencode(".jpg", img, p)
    assert ok
    return b.tobytes()


def pil_jpeg(img_bgr, q=90, subsampling=2, orientation=None, big_endian=False, **kw):
    from PIL import Image

    bio = io.BytesIO()
    args = dict(quality=q, subsampling=subsampling, **kw)
    if orientation is not None:
        args["exif"] = exif_block(orientation, big_endian)
    Image.fromarray(np.ascontiguousarray(img_bgr[:, :, ::-1])).save(bio, "JPEG", **args)
    return bio.getvalue()


def exif_block(orientation, big_endian=False):
    """'Exif\\0\\0' + a TIFF header and an IFD0 holding an unrelated tag and the orientation (SHORT, count 1)."""
    bo = "big" if big_endian else "little"
    t = (b"MM\x00*" if big_endian else b"II*\x00") + (8).to_bytes(4, bo) + (2).to_bytes(2, bo)
    t += (0x010F).to_bytes(2, bo) + (2).to_bytes(2, bo) + (4).to_bytes(4, bo) + b"abc\x00"  # Make, ASCII "abc"
    t += (0x0112).to_bytes(2, bo) + (3).to_bytes(2, bo) + (1).to_bytes(4, bo) + orientation.to_bytes(2, bo) + b"\x00\x00"
    t += (0).to_bytes(4, bo)
    return b"Exif\x00\x00" + t


def dqt16(b, scale=1):
    """The same file with every DQT rewritten with 16-bit entries (multiplied by `scale`)."""
    out, p = bytearray(b[:2]), 2
    while True:
        m, L = b[p + 1], (b[p + 2] << 8) | b[p + 3]
        seg = b[p:p + 2 + L]
        if m == 0xDB:
            s, i, body = seg[4:], 0, bytearray()
            while i < len(s):
                pq, tq = s[i] >> 4, s[i] & 15
                v = np.frombuffer(s[i + 1:i + 1 + 64 * (pq + 1)], np.uint8 if pq == 0 else ">u2").astype(np.int64)
                body += bytes([0x10 | tq]) + np.minimum(v * scale, 65535).astype(">u2").tobytes()
                i += 1 + 64 * (pq + 1)
            out += b"\xff\xdb" + (len(body) + 2).to_bytes(2, "big") + body
        else:
            out += seg
        p += 2 + L
        if m == 0xDA:
            return bytes(out + b[p:])


def corpus(large=False, seed=5):
    """-> list of (name, bytes) the GPU decoder accepts.  large=True adds 832x512, 1920x1080 and 4032x3024 frames."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in SMALL:
        for kind in ("flat", "noise", "check"):
            img = content(kind, h, w, rng)
            for q in (1, 50, 90, 100):
                for s in SAMPLINGS:
                    out.append(("%dx%d_%s_q%d_%s" % (w, h, kind, q, s), cv2_jpeg(img, q, s)))
                out.append(("%dx%d_%s_q%d_gray" % (w, h, kind, q), cv2_jpeg(img[:, :, 1].copy(), q)))
    img = content("noise", 37, 61, rng)
    for rst in (1, 7, 1000):
        for s in ("420", "444", "422"):
            out.append(("rst%d_%s" % (rst, s), cv2_jpeg(img, 90, s, rst=rst)))
    out.append(("rst7_gray", cv2_jpeg(img[:, :, 0].copy(), 90, rst=7)))
    for s in SAMPLINGS:
        out.append(("opt_%s" % s, cv2_jpeg(img, 90, s, optimize=True)))
    out.append(("dqt16_q50", dqt16(cv2_jpeg(img, 50, "420"))))
    out.append(("dqt16_x2_q90", dqt16(cv2_jpeg(img, 90, "444"), 2)))
    img2 = content("smooth", 40, 64, rng)
    for o in range(1, 9):
        out.append(("exif%d_le_420" % o, pil_jpeg(img2, 90, 2, o)))
        out.append(("exif%d_be_444" % o, pil_jpeg(img2, 75, 0, o, big_endian=True)))
    out.append(("pil_422_opt", pil_jpeg(img2, 85, 1, optimize=True)))
    if large:
        for h, w in ((512, 832), (1080, 1920)):
            big = content("smooth", h, w, rng)
            for s in SAMPLINGS:
                out.append(("%dx%d_smooth_q90_%s" % (w, h, s), cv2_jpeg(big, 90, s)))
            out.append(("%dx%d_smooth_q100_gray" % (w, h), cv2_jpeg(big[:, :, 0].copy(), 100)))
            out.append(("%dx%d_smooth_rst5_420" % (w, h), cv2_jpeg(big, 95, "420", rst=5)))
    return out


def large_frames(seed=9):
    """4032x3024 phone-camera-sized frames (noise and smooth, 4:2:0 / 4:4:4), and 1920x1080 noise."""
    rng = np.random.default_rng(seed)
    out = [("1920x1080_noise_q95_420", cv2_jpeg(content("noise", 1080, 1920, rng), 95, "420"))]
    out.append(("4032x3024_smooth_q90_420", cv2_jpeg(content("smooth", 3024, 4032, rng), 90, "420")))
    out.append(("4032x3024_noise_q90_444", cv2_jpeg(content("noise", 3024, 4032, rng), 90, "444")))
    out.append(("3024x4032_exif6_q90_420", pil_jpeg(content("smooth", 3024, 4032, rng), 90, 2, 6)))
    return out


def resize_edge_files(seed=12):
    """Files whose frames hit the resizer's edges at an 832x512 input: the 1x1, 7x5 and 17x9 (w x h) corpus files
    (up-scaling from 1-pixel sides), a 1663x1024 frame (exact 1/2 scale, last column cut) and an EXIF-6 file stored
    1023x1664 whose displayed frame is 1664x1023 (last row cut)."""
    rng = np.random.default_rng(seed)
    out = [(n, b) for n, b in corpus() if n.split("_")[0] in ("1x1", "7x5", "17x9")]
    out.append(("1663x1024_noise_q90_420", cv2_jpeg(content("noise", 1024, 1663, rng), 90, "420")))
    out.append(("exif6_1664x1023_q90_420", pil_jpeg(content("noise", 1664, 1023, rng), 90, 2, 6)))
    return out


def not_decoded(seed=6):
    """-> list of (name, bytes) the decoder must leave to cv2: progressive, CMYK, 4:1:1, PNG, RGB (Adobe transform 0)."""
    import cv2
    from PIL import Image

    rng = np.random.default_rng(seed)
    img = content("noise", 37, 61, rng)
    out = []
    bio = io.BytesIO()
    Image.fromarray(img).save(bio, "JPEG", progressive=True, quality=90)
    out.append(("progressive", bio.getvalue()))
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    out.append(("progressive_cv2", b.tobytes()))
    bio = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(bio, "JPEG", quality=90)
    out.append(("cmyk", bio.getvalue()))
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111])
    out.append(("411", b.tobytes()))
    out.append(("png", cv2.imencode(".png", img)[1].tobytes()))
    bio = io.BytesIO()
    Image.fromarray(img).save(bio, "JPEG", quality=90, subsampling=0, keep_rgb=True)
    out.append(("rgb", bio.getvalue()))
    return out


def scan_start(b):
    """Offset of the first entropy-coded byte (after the SOS header)."""
    p = 2
    while True:
        m, L = b[p + 1], (b[p + 2] << 8) | b[p + 3]
        p += 2 + L
        if m == 0xDA:
            return p


def damaged(seed=7):
    """A fixed, small set of truncated and corrupted files: cuts inside the headers and the scan, flipped scan bytes, a
    wrong restart marker."""
    rng = np.random.default_rng(seed)
    img = content("noise", 37, 61, rng)
    base = [cv2_jpeg(img, 90, "420"), cv2_jpeg(img, 75, "444", rst=3), cv2_jpeg(content("smooth", 64, 96, rng), 90, "422")]
    out = []
    for k, b in enumerate(base):
        s0 = scan_start(b)
        for cut in (3, 20, s0 - 5, s0 + 2, (s0 + len(b)) // 2, len(b) - 2, len(b) - 1):
            out.append(("cut%d_%d" % (k, cut), b[:cut]))
        for j, pos in enumerate(rng.integers(s0, len(b) - 2, 6)):
            c = bytearray(b)
            c[pos] ^= int(rng.integers(1, 256))
            out.append(("flip%d_%d" % (k, j), bytes(c)))
    b = base[1]
    i = b.find(b"\xff\xd1", scan_start(b))
    c = bytearray(b)
    c[i + 1] = 0xD5
    out.append(("rst_out_of_sequence", bytes(c)))
    return out
