"""Seeded corpus of the JPEG frames SMAPB_JPEG_COLOUR adds (tests/test_jpeg_colour_cpu.py, tests/test_jpeg_colour_gpu.py),
built at test time: CMYK files Pillow writes (ids C, M, Y, K with the factors on C, Adobe transform 0) at its three
subsamplings and the same relabelled YCCK, RGB files Pillow writes with keep_rgb (Adobe transform 0), cv2's 4:1:1, and
files written from coefficients here - YCCK
(Adobe transform 2), RGB marked only by its 'R','G','B' ids, 4:1:1, 4:1:0, factors of 3, luma coarser than chroma, mixed
chroma factors, exactly 10 blocks per MCU, with restart intervals, EXIF orientations and partial MCUs, sequential and
progressive (jpeg_scans' scripts) - and the frames cv2 and the decoder both refuse: fractional sampling ratios, 11 blocks
per MCU, 2 components.

corpus() -> [(name, bytes, expect)]: expect is DECODE (equal to cv2.imdecode) or the status smapb_jpeg_info_ex(SMAPB_JPEG_SCANS
| SMAPB_JPEG_COLOUR) refuses the file with."""
import io

import numpy as np

from jpeg_corpus import SMALL, content, exif_block
from jpeg_scans import SCRIPTS, SEQUENTIAL, _codes, _optimal_table, _scan_tokens, _Writer
from jpeg_writer import _marker
from oracle import jpeg_numpy as J

DECODE = "decode"
JFIF = _marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")


def adobe(transform):
    """APP14 'Adobe' (version 100, flags 0, 0) with the transform flag."""
    return _marker(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00" + bytes([transform]))


def exif(orientation):
    return _marker(0xE1, exif_block(orientation))


# ---- Pillow --------------------------------------------------------------------------------------------------------------
def cmyk_of(img_bgr, rng):
    """A CMYK image from a BGR one: the inks of R, G, B and a K plane of its own."""
    k = np.clip(img_bgr.mean(2) + rng.integers(-40, 41, img_bgr.shape[:2]), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(np.concatenate([255 - img_bgr[:, :, ::-1], k[:, :, None]], 2))


def pil_cmyk(cmyk, q=90, subsampling=0, orientation=None, **kw):
    from PIL import Image

    bio = io.BytesIO()
    args = dict(quality=q, subsampling=subsampling, **kw)
    if orientation is not None:
        args["exif"] = exif_block(orientation)
    Image.fromarray(cmyk, "CMYK").save(bio, "JPEG", **args)
    return bio.getvalue()


def ycck_of(b):
    """The same coefficients relabelled YCCK: the file's Adobe APP14 transform flag set to 2."""
    i = b.find(b"\xff\xee")
    assert i > 0 and b[i + 4:i + 9] == b"Adobe"
    return b[:i + 15] + b"\x02" + b[i + 16:]


def cv2_411(img_bgr, q=90):
    """4:1:1 (luma 4x1) as libjpeg writes it."""
    import cv2

    ok, b = cv2.imencode(".jpg", img_bgr, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])
    assert ok
    return b.tobytes()


def pil_rgb(img_bgr, q=90, **kw):
    """keep_rgb: Pillow writes 4:4:4 only"""
    from PIL import Image

    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img_bgr[:, :, ::-1])).save(bio, "JPEG", quality=q, keep_rgb=True, **kw)
    return bio.getvalue()


# ---- coefficient-level writer ------------------------------------------------------------------------------------------
def header(h, w, comps):
    """comps [(id, H, V)] -> the hd dict jpeg_scans' tokeniser reads (the frame geometry of the decoder)."""
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    if len(comps) == 1:
        comps, hmax, vmax = [(comps[0][0], 1, 1)], 1, 1
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    return dict(h=h, w=w, comps=[c + (0,) for c in comps], hmax=hmax, vmax=vmax, mcux=mcux, mcuy=mcuy, nmcu=mcux * mcuy)


def random_coef(rng, hd, ac=12, amp=60):
    """int [nmcu * blocks per MCU, 64]: every block at a random level (DC at q = 1) with `ac` random low-frequency
    coefficients, so neighbouring blocks differ and every upsampling filter has edges to blend."""
    bpm = sum(c[1] * c[2] for c in hd["comps"])
    n = hd["nmcu"] * bpm
    c = np.zeros((n, 64), np.int64)
    c[:, 0] = rng.integers(-1020, 1021, n)
    c[:, J.ZIGZAG[1:1 + ac]] = rng.integers(-amp, amp + 1, (n, ac))
    return c


def write(coef, h, w, comps, markers=(), script=None, progressive=False, dri=0, sof_comps=None):
    """-> a JPEG file coding `coef` (frame-MCU layout of oracle/jpeg_numpy.py) for frame components comps [(id, H, V)]
    with q = 1 (one DQT, id 0) and libjpeg's optimal tables per scan.  script: [(components, Ss, Se, Ah, Al)], default
    one interleaved sequential scan of every component; progressive: SOF2 instead of SOF0; markers: raw segments after
    SOI; sof_comps: the (id, H, V) written in the SOF when they differ from the coded geometry (a refused frame)."""
    hd = header(h, w, comps)
    script = script or [(tuple(range(len(comps))), 0, 63, 0, 0)]
    out = bytearray(b"\xff\xd8")
    for m in markers:
        out += m
    out += _marker(0xDB, bytes([0]) + bytes([1] * 64))
    body = bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([len(comps)])
    for cid, hs, vs in sof_comps or comps:
        body += bytes([cid, (hs << 4) | vs, 0])
    out += _marker(0xC2 if progressive else 0xC0, body)
    if dri:
        out += _marker(0xDD, dri.to_bytes(2, "big"))
    for sc, ss, se, ah, al in script:
        toks = _scan_tokens(coef, hd, sc, ss, se, ah, al, dri)
        tables, dht = {}, bytearray()
        for key in sorted({t[1] for t in toks if t[0] == "s"}):
            freq = [0] * 256
            for t in toks:
                if t[0] == "s" and t[1] == key:
                    freq[t[2]] += 1
            counts, syms = _optimal_table(freq)
            tables[key] = _codes(counts, syms)
            dht += bytes([(0 if key[0] == "dc" else 0x10) | key[1]]) + bytes(counts) + bytes(syms)
        if dht:
            out += _marker(0xC4, dht)
        sos = bytes([len(sc)]) + b"".join(bytes([comps[c][0], (k << 4) | k]) for k, c in enumerate(sc))
        out += _marker(0xDA, sos + bytes([ss, se, (ah << 4) | al]))
        wr, rst = _Writer(), 0
        for t in toks:
            if t[0] == "s":
                wr.bits(*tables[t[1]][t[2]])
            elif t[0] == "b":
                wr.bits(t[1], t[2])
            else:
                wr.flush()
                wr.out += bytes([0xFF, 0xD0 + rst % 8])
                rst += 1
        wr.flush()
        out += wr.out
    return bytes(out + b"\xff\xd9")


def script_for(name, nf):
    """jpeg_scans' script for 3 components, on nf components: a 4th component takes the scans of the 3rd (in the same
    interleaved scan, or a scan of its own right after), so a 4-component frame gets the same progression."""
    out = []
    for comps, ss, se, ah, al in SCRIPTS[name]:
        c = tuple(x for x in comps if x < nf)
        if nf == 4 and 2 in comps and len(comps) > 1:
            c += (3,)
        if c:
            out.append((c, ss, se, ah, al))
        if nf == 4 and comps == (2,):
            out.append(((3,), ss, se, ah, al))
    return out


# name -> (components [(id, H, V)], marker segments)
YCC = (1, 2, 3)
FRAMES = {
    "ycck_444": ([(1, 1, 1), (2, 1, 1), (3, 1, 1), (4, 1, 1)], [adobe(2)]),
    "ycck_420": ([(1, 2, 2), (2, 1, 1), (3, 1, 1), (4, 2, 2)], [adobe(2)]),
    "cmyk_c22": ([(67, 2, 2), (77, 1, 1), (89, 1, 1), (75, 1, 1)], [adobe(0)]),
    "cmyk_plain_mixed": ([(1, 2, 1), (2, 1, 1), (3, 2, 1), (4, 1, 1)], []),
    "rgb_ids": ([(82, 1, 1), (71, 1, 1), (66, 1, 1)], []),
    "rgb_ids_422": ([(82, 2, 1), (71, 1, 1), (66, 1, 1)], []),
    "rgb_adobe": ([(1, 1, 1), (2, 1, 1), (3, 1, 1)], [adobe(0)]),
    "ycc_411": ([(1, 4, 1), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "ycc_410": ([(1, 4, 2), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "ycc_31": ([(1, 3, 1), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "ycc_13": ([(1, 1, 3), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "ycc_32": ([(1, 3, 2), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "ycc_luma_coarse": ([(1, 1, 1), (2, 2, 2), (3, 2, 2)], [JFIF]),
    "ycc_luma_h1v2": ([(1, 1, 1), (2, 1, 2), (3, 1, 1)], [JFIF]),
    "ycc_mixed_h": ([(1, 4, 1), (2, 2, 1), (3, 1, 1)], [JFIF]),
    "ycc_mixed_v": ([(1, 2, 2), (2, 1, 2), (3, 1, 1)], [JFIF]),
    "ycc_mixed_hv": ([(1, 2, 2), (2, 2, 1), (3, 1, 2)], [JFIF]),
    "ycc_14": ([(1, 1, 4), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "blocks10_ycc": ([(1, 2, 2), (2, 2, 2), (3, 2, 1)], [JFIF]),
    "blocks10_ycck": ([(1, 2, 2), (2, 2, 2), (3, 1, 1), (4, 1, 1)], [adobe(2)]),
    "gray_factor_4x4": ([(1, 4, 4)], []),
}
# frames cv2 refuses too
REFUSED = {
    "fractional_h": ([(1, 3, 1), (2, 2, 1), (3, 1, 1)], [JFIF]),
    "fractional_v": ([(1, 2, 3), (2, 1, 2), (3, 1, 1)], [JFIF]),
    "blocks11": ([(1, 3, 3), (2, 1, 1), (3, 1, 1)], [JFIF]),
    "blocks11_cmyk": ([(1, 2, 2), (2, 2, 2), (3, 2, 1), (4, 1, 1)], [adobe(0)]),
    "two_components": ([(1, 1, 1), (2, 1, 1)], []),
}
PROGRESSIVE = ("libjpeg", "spectral_only", "approximation_deep", "seq_per_component")


def coefficient_files(seed=51):
    """-> [(name, bytes, expect)] written from coefficients."""
    rng = np.random.default_rng(seed)
    out = []
    for name, (comps, marks) in FRAMES.items():
        for h, w in ((1, 1), (9, 17), (37, 61), (70, 45)):
            hd = header(h, w, comps)
            coef = random_coef(rng, hd)
            out.append(("%s_%dx%d" % (name, h, w), write(coef, h, w, comps, marks), DECODE))
        hd = header(37, 61, comps)
        coef = random_coef(rng, hd)
        out.append((name + "_rst3_exif6", write(coef, 37, 61, comps, list(marks) + [exif(6)], dri=3), DECODE))
        if len(comps) > 1:
            for s in PROGRESSIVE:
                out.append(("%s_%s" % (name, s), write(coef, 37, 61, comps, marks, script_for(s, len(comps)),
                                                       s not in SEQUENTIAL), DECODE))
            out.append((name + "_libjpeg_rst2_exif3", write(coef, 37, 61, comps, list(marks) + [exif(3)],
                                                            script_for("libjpeg", len(comps)), True, dri=2), DECODE))
    for name, (comps, marks) in REFUSED.items():
        # coded as a frame the tokeniser can lay out; the SOF declares the refused geometry
        coded = [(c[0], 1, 1) for c in comps]
        hd = header(16, 24, coded)
        out.append((name, write(random_coef(rng, hd), 16, 24, coded, marks, sof_comps=comps), J.UNSUPPORTED))
    # Adobe transforms libjpeg only warns about, on 4 components
    comps = FRAMES["ycck_444"][0]
    coef = random_coef(rng, header(16, 24, comps))
    for t in (1, 3):
        out.append(("adobe%d_cmyk" % t, write(coef, 16, 24, comps, [adobe(t)]), J.UNSUPPORTED))
    return out


def encoded_files(seed=53):
    """-> [(name, bytes, expect)]: Pillow's CMYK at subsampling 0 / 1 / 2 (and relabelled YCCK) and RGB (keep_rgb), with
    and without EXIF, and cv2's 4:1:1."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in SMALL + [(70, 45)]:
        for kind in ("noise", "smooth"):
            img = content(kind, h, w, rng)
            for sub in (0, 1, 2):
                out.append(("pil_cmyk%d_%s_%dx%d" % (sub, kind, h, w), pil_cmyk(cmyk_of(img, rng), 90, sub), DECODE))
            out.append(("pil_rgb_%s_%dx%d" % (kind, h, w), pil_rgb(img, 90), DECODE))
            out.append(("pil_ycck2_%s_%dx%d" % (kind, h, w), ycck_of(pil_cmyk(cmyk_of(img, rng), 90, 2)), DECODE))
            out.append(("cv2_411_%s_%dx%d" % (kind, h, w), cv2_411(img), DECODE))
    img = content("smooth", 37, 61, rng)
    for o in (3, 6, 8):
        out.append(("pil_cmyk2_exif%d" % o, pil_cmyk(cmyk_of(img, rng), 90, 2, o), DECODE))
    out.append(("pil_cmyk2_progressive", pil_cmyk(cmyk_of(img, rng), 90, 2, progressive=True), DECODE))
    out.append(("pil_rgb_progressive", pil_rgb(img, 90, progressive=True), DECODE))
    return out


def corpus():
    return encoded_files() + coefficient_files()


LARGE_KINDS = ("cmyk444", "cmyk420", "ycck420", "ycc411")


def large_frames(kind, h, w, n=1, seed=57):
    """n seeded h x w frames (smooth content, q90) of one of LARGE_KINDS: Pillow's CMYK at subsampling 0 or 2, the 4:2:0
    one relabelled YCCK, or cv2's 4:1:1."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        img = content("smooth", h, w, rng)
        if kind == "ycc411":
            out.append(cv2_411(img))
            continue
        b = pil_cmyk(cmyk_of(img, rng), 90, 0 if kind == "cmyk444" else 2)
        out.append(ycck_of(b) if kind == "ycck420" else b)
    return out
