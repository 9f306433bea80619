"""CPU restatement of the frames SMAPB_JPEG_COLOUR adds to the GPU JPEG decoder (smap_b200/csrc/jpeg.cu): CMYK, YCCK and
RGB frames and every integral sampling, with SMAPB_JPEG_SCANS (single-scan, multi-scan sequential and progressive
files).  The entropy decoding is jpeg_scans_numpy's and the IDCT jpeg_numpy's, both generic in the blocks of an MCU; what
is restated here is the header walk's wider acceptance, libjpeg-turbo 3.x's choice of upsampling method per component and
the conversion to BGR that cv2.imread(path, IMREAD_COLOR) applies for each colour space.

    hd = parse(data)                  # jpeg_parse's rules with SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR; NotDecoded otherwise
    bgr = colour(J.idct_planes(S.entropy_decode(data, hd), hd), hd)
    decode(data) does all three.

Colour spaces follow libjpeg's default_decompress_parms; upsampling its jinit_upsampler (a component whose factors equal
the frame's maxima is used as is, one at half the width and / or half the height takes the triangle filters jpeg_numpy
restates, every other integral ratio is replicated); CMYK and YCCK frames are decoded by libjpeg to CMYK (YCCK through the
YCbCr tables, C = 255 - R and so on) and converted by cv2 with K - ((255 - ink) * K >> 8) per ink.
"""
import numpy as np

from . import jpeg_numpy as J
from . import jpeg_scans_numpy as S
from .jpeg_numpy import CORRUPT, MALFORMED, OK, TOO_LARGE, UNSUPPORTED, NotDecoded

MAX_BLOCKS = 10  # libjpeg's D_MAX_BLOCKS_IN_MCU
GRAY, YCC, RGB, CMYK, YCCK = "gray", "ycc", "rgb", "cmyk", "ycck"


def colour_space(nf, ids, jfif, adobe, adobe_transform):
    """libjpeg's rule -> one of GRAY, YCC, RGB, CMYK, YCCK; None for the 4-component Adobe transforms libjpeg only warns
    about."""
    if nf == 1:
        return GRAY
    if nf == 3:
        if jfif:
            return YCC
        if adobe:
            return YCC if adobe_transform != 0 else RGB
        return RGB if tuple(ids) == (82, 71, 66) else YCC
    if not adobe or adobe_transform == 0:
        return CMYK
    return YCCK if adobe_transform == 2 else None


def _sampling(comps):
    """Factors 1..4, integral ratios to the maxima, at most MAX_BLOCKS blocks per MCU; -> comps as the decoder uses them."""
    if any(not (1 <= c[1] <= 4 and 1 <= c[2] <= 4) for c in comps):
        raise NotDecoded(UNSUPPORTED, "sampling factor outside 1..4")
    if len(comps) == 1:
        return [(comps[0][0], 1, 1, comps[0][3])]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    if any(hmax % c[1] or vmax % c[2] for c in comps):
        raise NotDecoded(UNSUPPORTED, "fractional sampling")
    if sum(c[1] * c[2] for c in comps) > MAX_BLOCKS:
        raise NotDecoded(UNSUPPORTED, "more than %d blocks per MCU" % MAX_BLOCKS)
    return comps


def parse(data):
    """The marker walk of jpeg_scans_numpy.parse with SMAPB_JPEG_COLOUR's frames.  -> the same dict plus 'colour'."""
    d = bytes(data)
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise NotDecoded(MALFORMED, "no SOI")
    p = 2
    qt, qt_used, dht, latched = [None] * 4, [False] * 4, {}, {}
    dri, sof, progressive = 0, None, False
    jfif = adobe = False
    adobe_transform, orientation = 0, None
    coef_bits = nscanned = None
    scans = []
    while True:
        if p + 2 > n or d[p] != 0xFF:
            raise NotDecoded(MALFORMED, "marker expected at %d" % p)
        while p + 1 < n and d[p + 1] == 0xFF:
            p += 1
        if p + 2 > n:
            raise NotDecoded(MALFORMED, "truncated marker")
        m = d[p + 1]
        p += 2
        if m == 0xD9:
            if not scans:
                raise NotDecoded(MALFORMED, "EOI before a scan")
            break
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise NotDecoded(MALFORMED, "marker %02X out of place" % m)
        if p + 2 > n:
            raise NotDecoded(MALFORMED, "truncated length")
        L = J._u16(d, p)
        if L < 2 or p + L > n:
            raise NotDecoded(MALFORMED, "segment length")
        s = d[p + 2:p + L]
        p += L
        if m == 0xDB:
            i = 0
            while i < len(s):
                pq, tq = s[i] >> 4, s[i] & 15
                if pq > 1 or tq > 3 or i + 1 + 64 * (pq + 1) > len(s):
                    raise NotDecoded(MALFORMED, "DQT")
                if qt_used[tq]:
                    raise NotDecoded(UNSUPPORTED, "DQT redefines a table a scan used")
                q = np.zeros(64, np.int64)
                q[J.ZIGZAG] = np.frombuffer(s, np.uint8 if pq == 0 else ">u2", 64, i + 1).astype(np.int64)
                qt[tq] = q
                i += 1 + 64 * (pq + 1)
        elif m == 0xC4:
            i = 0
            while i < len(s):
                if i + 17 > len(s):
                    raise NotDecoded(MALFORMED, "DHT")
                tc, th = s[i] >> 4, s[i] & 15
                counts = list(s[i + 1:i + 17])
                tot = sum(counts)
                if tc > 1 or th > 3 or tot > 256 or i + 17 + tot > len(s):
                    raise NotDecoded(MALFORMED, "DHT")
                dht[(tc, th)] = (counts, list(s[i + 17:i + 17 + tot]))
                i += 17 + tot
        elif m == 0xDD:
            if len(s) != 2:
                raise NotDecoded(MALFORMED, "DRI")
            dri = J._u16(s, 0)
        elif m in (0xC0, 0xC1, 0xC2):
            if sof is not None or len(s) < 6:
                raise NotDecoded(MALFORMED, "SOF")
            progressive = m == 0xC2
            prec, hh, ww, nf = s[0], J._u16(s, 1), J._u16(s, 3), s[5]
            if len(s) != 6 + 3 * nf:
                raise NotDecoded(MALFORMED, "SOF length")
            if prec != 8 or hh == 0 or ww == 0 or nf not in (1, 3, 4):
                raise NotDecoded(UNSUPPORTED, "precision / size / components")
            comps = [(s[6 + 3 * c], s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]) for c in range(nf)]
            for c in range(nf):
                if comps[c][3] > 3 or any(comps[e][0] == comps[c][0] for e in range(c)):
                    raise NotDecoded(MALFORMED, "component ids / table ids")
            comps = _sampling(comps)
            if hh * ww > J.MAX_PIXELS:
                raise NotDecoded(TOO_LARGE, "over the pixel cap")
            hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
            mcux, mcuy = -(-ww // (8 * hmax)), -(-hh // (8 * vmax))
            sof = (hh, ww, comps)
            coef_bits = [[-1] * 64 for _ in range(nf)]
            nscanned = [0] * nf
        elif 0xC3 <= m <= 0xCF:
            raise NotDecoded(UNSUPPORTED, "SOF%d / DAC / JPG" % (m - 0xC0))
        elif m in (0xE0, 0xE1, 0xEE):
            if scans:
                raise NotDecoded(UNSUPPORTED, "APP0 / APP1 / APP14 after a scan")
            if m == 0xE0 and len(s) >= 14 and s[:5] == b"JFIF\x00":
                jfif = True
            elif m == 0xEE and len(s) >= 12 and s[:5] == b"Adobe":
                adobe, adobe_transform = True, s[11]
            elif m == 0xE1:
                o = J._exif_orientation(s)
                if o is not None:
                    if orientation is not None:
                        raise NotDecoded(UNSUPPORTED, "two EXIF blocks")
                    orientation = o
        elif 0xE2 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            if sof is None:
                raise NotDecoded(MALFORMED, "SOS before SOF")
            if len(scans) == S.MAX_SCANS:
                raise NotDecoded(UNSUPPORTED, "more than %d scans" % S.MAX_SCANS)
            hh, ww, comps = sof
            nf = len(comps)
            ns = s[0] if len(s) >= 1 else 0
            if ns < 1 or ns > nf or len(s) != 4 + 2 * ns:
                raise NotDecoded(MALFORMED, "SOS length")
            ss, se, ah, al = s[1 + 2 * ns], s[2 + 2 * ns], s[3 + 2 * ns] >> 4, s[3 + 2 * ns] & 15
            ids = [c[0] for c in comps]
            sc = []
            for k in range(ns):
                if s[1 + 2 * k] not in ids:
                    raise NotDecoded(UNSUPPORTED, "unknown component")
                c = ids.index(s[1 + 2 * k])
                if sc and c <= sc[-1]:
                    raise NotDecoded(UNSUPPORTED, "scan components not in frame order")
                sc.append(c)
            if not progressive:
                if (ss, se, ah, al) != (0, 63, 0, 0):
                    raise NotDecoded(UNSUPPORTED, "Ss/Se/Ah/Al of a sequential scan")
                for c in sc:
                    if nscanned[c]:
                        raise NotDecoded(UNSUPPORTED, "component in two sequential scans")
                    nscanned[c] += 1
            else:
                if (se != 0) if ss == 0 else (ss > se or se > 63 or ns != 1):
                    raise NotDecoded(UNSUPPORTED, "bad spectral selection")
                if (ah != 0 and al != ah - 1) or al > 13:
                    raise NotDecoded(UNSUPPORTED, "bad successive approximation")
                for c in sc:
                    cb = coef_bits[c]
                    if ss > 0 and cb[0] < 0:
                        raise NotDecoded(UNSUPPORTED, "AC before DC")
                    for i in range(ss, se + 1):
                        if ah != max(cb[i], 0):
                            raise NotDecoded(UNSUPPORTED, "bogus progression")
                        cb[i] = al
            dc_first, uses_ac = ss == 0 and ah == 0, se > 0
            dcs, acs = [], []
            for k, c in enumerate(sc):
                td, ta = s[2 + 2 * k] >> 4, s[2 + 2 * k] & 15
                dcs.append(None)
                acs.append(None)
                if dc_first:
                    if (0, td) not in dht:
                        raise NotDecoded(UNSUPPORTED, "table not defined")
                    if any(v > 15 for v in dht[(0, td)][1]):
                        raise NotDecoded(MALFORMED, "DC symbol > 15")
                    J._check_canonical(dht[(0, td)][0])
                    dcs[-1] = dht[(0, td)]
                if uses_ac:
                    if (1, ta) not in dht:
                        raise NotDecoded(UNSUPPORTED, "table not defined")
                    J._check_canonical(dht[(1, ta)][0])
                    acs[-1] = dht[(1, ta)]
                if c not in latched:
                    q = qt[comps[c][3]]
                    if q is None:
                        raise NotDecoded(UNSUPPORTED, "quantiser not defined")
                    if q.max() > 32767:
                        raise NotDecoded(UNSUPPORTED, "quantiser above 32767")
                    latched[c] = q
                    qt_used[comps[c][3]] = True
            if ns == 1:
                c = sc[0]
                cw, ch = -(-ww * comps[c][1] // hmax), -(-hh * comps[c][2] // vmax)
                smx, snmcu, sbpm = -(-cw // 8), -(-cw // 8) * -(-ch // 8), 1
            else:
                smx, snmcu, sbpm = mcux, mcux * mcuy, sum(comps[c][1] * comps[c][2] for c in sc)
            nseg = -(-snmcu // dri) if dri else 1
            segs = []
            start = q = p
            while True:
                q = d.find(b"\xff", q)
                if q < 0 or q + 1 >= n:
                    raise NotDecoded(MALFORMED, "no marker after the scan")
                mk = d[q + 1]
                if mk == 0:
                    q += 2
                    continue
                rst = 0xD0 <= mk <= 0xD7
                if rst and (not dri or mk - 0xD0 != len(segs) % 8 or len(segs) + 1 >= nseg):
                    raise NotDecoded(CORRUPT, "restart marker out of sequence")
                segs.append((start, q))
                if not rst:
                    break
                start = q = q + 2
            if len(segs) != nseg:
                raise NotDecoded(CORRUPT, "%d restart segments, %d expected" % (len(segs), nseg))
            if segs[-1][1] - segs[0][0] > S.MAX_SCAN_BYTES:
                raise NotDecoded(TOO_LARGE, "scan over 2^28 bytes")
            scans.append(dict(comps=sc, ss=ss, se=se, ah=ah, al=al, dri=dri, mcux=smx, nmcu=snmcu, bpm=sbpm, segments=segs,
                              dc=dcs, ac=acs))
            p = q
        else:
            raise NotDecoded(UNSUPPORTED, "marker %02X" % m)
    hh, ww, comps = sof
    nf = len(comps)
    for c in range(nf):
        if not progressive:
            if nscanned[c] != 1:
                raise NotDecoded(UNSUPPORTED, "component not in exactly one scan")
            continue
        if coef_bits[c][0] < 0:
            raise NotDecoded(UNSUPPORTED, "component without DC")
        if any(b != 0 for b in coef_bits[c][1:S.SAVED_COEFS]):
            raise NotDecoded(UNSUPPORTED, "coefficient 1..9 not fully refined: libjpeg-turbo smooths the output")
    cs = colour_space(nf, [c[0] for c in comps], jfif, adobe, adobe_transform)
    if cs is None:
        raise NotDecoded(UNSUPPORTED, "Adobe transform %d with 4 components" % adobe_transform)
    H, W = (ww, hh) if orientation and orientation >= 5 else (hh, ww)
    return dict(h=hh, w=ww, out_h=H, out_w=W, orientation=orientation or 1, comps=comps, hmax=hmax, vmax=vmax, mcux=mcux,
                mcuy=mcuy, nmcu=mcux * mcuy, qt=[latched[c] for c in range(nf)], scans=scans, progressive=progressive,
                colour=cs)


def info(data):
    """-> (status, out_h, out_w, orientation): what smapb_jpeg_info_ex(SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR) reports."""
    try:
        hd = parse(data)
    except NotDecoded as e:
        return e.status, 0, 0, 0
    return OK, hd["out_h"], hd["out_w"], hd["orientation"]


def upsample(plane, hs, vs, hmax, vmax, H, W):
    """A component plane (padded) at factors (hs, vs) -> int plane [H, W] at the frame's (hmax, vmax), by the method
    libjpeg-turbo picks: ratios of 1 and 2 are jpeg_numpy's (as is, fancy h2v1 / h1v2 / h2v2, replication when a
    halved width is 2 samples or less), any other integral ratio replication."""
    rh, rv = hmax // hs, vmax // vs
    if rh <= 2 and rv <= 2:
        return J.upsample(plane, 1, 1, H, W, rh, rv)
    cw, ch = -(-W // rh), -(-H // rv)
    return np.repeat(np.repeat(plane[:ch, :cw].astype(np.int64), rv, 0), rh, 1)[:H, :W]


def _ycc_rgb(y, cb, cr):
    cb, cr, half = cb - 128, cr - 128, 1 << 15
    r = y + ((91881 * cr + half) >> 16)
    g = y + ((-46802 * cr - 22554 * cb + half) >> 16)
    b = y + ((116130 * cb + half) >> 16)
    return [np.clip(v, 0, 255) for v in (r, g, b)]


def _ink(x, k):
    """cv2's CMYK -> BGR of one ink (icvCvt_CMYK2BGR_8u_C4C3R)."""
    return k - (((255 - x) * k) >> 8)


def colour(planes, hd):
    H, W = hd["h"], hd["w"]
    up = [upsample(p, c[1], c[2], hd["hmax"], hd["vmax"], H, W) for p, c in zip(planes, hd["comps"])]
    cs = hd["colour"]
    if cs == GRAY:
        r = g = b = up[0]
    elif cs == RGB:
        r, g, b = up
    elif cs == CMYK:
        r, g, b = (_ink(x, up[3]) for x in up[:3])
    else:
        r, g, b = _ycc_rgb(*up[:3])
        if cs == YCCK:
            r, g, b = (_ink(255 - x, up[3]) for x in (r, g, b))
    return J.orient(np.stack([b, g, r], 2).astype(np.uint8), hd["orientation"])


def decode(data):
    """-> uint8 BGR [H, W, 3] as cv2.imread(path, IMREAD_COLOR) returns it; NotDecoded for inputs left to cv2."""
    hd = parse(data)
    return colour(J.idct_planes(S.entropy_decode(data, hd), hd), hd)
