"""CPU restatement of the GPU JPEG decoder (smap_b200/csrc/jpeg.cu), pinned byte for byte against cv2.imread(path, IMREAD_COLOR)
(opencv-python's bundled libjpeg-turbo) by tests/test_jpeg_cpu.py, as preprocess_numpy.py is pinned against cv2.resize.

Same inputs, same acceptance rules and the same arithmetic as the library, stage by stage, so a GPU test can compare
coefficients and planes and name the stage that disagrees:

    hdr = parse(data)                  # marker walk, tables, restart segments, EXIF orientation; NotDecoded otherwise
    coef = entropy_decode(data, hdr)   # sequential Huffman decoding -> int16 [blocks, 64] (natural order, DC absolute)
    planes = idct_planes(coef, hdr)    # dequantisation + accurate-integer IDCT, one uint8 plane per component
    bgr = colour(planes, hdr)          # fancy upsampling, YCbCr -> BGR, EXIF orientation
    decode(data) does all four.

The arithmetic restated here is the published one: ITU-T T.81 (Huffman decoding, DC prediction, restart intervals), the
Loeffler-Ligtenberg-Moschytz 8-point IDCT in the 13-bit fixed point with 2 extra pass-1 bits that the IJG documents for its
"accurate integer" method, the triangle ("fancy") upsampling filters and the JFIF YCbCr -> RGB equations with 16-bit
fixed-point constants.  Which of two range-limiting conventions cv2's build applies after the IDCT (saturation, or a
10-bit wrap-around table) was decided by decoding q100 checkerboards: saturation (IDCT_CLAMP).
"""
import numpy as np

# status codes (include/smap_b200.h, SMAPB_JPEG_*)
OK, UNSUPPORTED, MALFORMED, CORRUPT, TOO_LARGE = 0, 1, 2, 3, 4
MAX_PIXELS = 1 << 26  # SMAPB_JPEG_MAX_PIXELS

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63])
IDCT_CLAMP = True  # saturate the IDCT output to 0..255 (False: index a 10-bit wrap-around range table)
# cv2's IDCT works on 16-bit lanes (dequantised coefficients, pass-1 outputs, sums of up to four of them).  While every
# dequantised coefficient and every pass-1 output stays within +-GUARD, none of those lanes overflows and the result is the
# exact fixed-point IDCT restated here; blocks beyond it (16-bit quantisers far above what an encoder writes, corrupt data)
# are left to cv2.
GUARD = 8191


class NotDecoded(Exception):
    def __init__(self, status, why):
        super().__init__(why)
        self.status = status


def _u16(d, i):
    return (d[i] << 8) | d[i + 1]


def _huff_table(counts, symbols):
    """Canonical code assignment (T.81 Annex C) -> list of 65536 entries (len << 8 | symbol) indexed by the next 16 bits;
    0 = no code.  Tables that are over-subscribed or use a code of all ones are rejected (_check_canonical)."""
    lut = [0] * 65536
    code, k = 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            if code >= (1 << length) - 1:
                raise NotDecoded(MALFORMED, "over-subscribed Huffman table or a code of all ones")
            lo = code << (16 - length)
            e = (length << 8) | symbols[k]
            for j in range(lo, lo + (1 << (16 - length))):
                lut[j] = e
            code += 1
            k += 1
        code <<= 1
    return lut


def _check_canonical(counts):
    """libjpeg's rule (jpeg_make_d_derived_tbl): the codes of each length must fit it, and none may be all ones, so a
    complete code is refused too."""
    code = 0
    for length in range(1, 17):
        code += counts[length - 1]
        if code >= (1 << length):
            raise NotDecoded(MALFORMED, "over-subscribed Huffman table or a code of all ones")
        code <<= 1


def _exif_orientation(seg):
    """seg: APP1 payload.  -> orientation 1..8; NotDecoded for an EXIF block whose orientation is not clean."""
    if len(seg) < 6 or seg[:6] != b"Exif\x00\x00":
        return None
    t = seg[6:]
    if len(t) < 8:
        raise NotDecoded(UNSUPPORTED, "short TIFF header")
    if t[:4] == b"II*\x00":
        le = True
    elif t[:4] == b"MM\x00*":
        le = False
    else:
        raise NotDecoded(UNSUPPORTED, "bad TIFF header")

    def rd(i, n):
        if i < 0 or i + n > len(t):
            raise NotDecoded(UNSUPPORTED, "EXIF offset out of range")
        return int.from_bytes(t[i:i + n], "little" if le else "big")

    ifd = rd(4, 4)
    n = rd(ifd, 2)
    for e in range(n):
        p = ifd + 2 + 12 * e
        if rd(p, 2) == 0x0112:
            typ, cnt, val = rd(p + 2, 2), rd(p + 4, 4), rd(p + 8, 2)
            if typ != 3 or cnt != 1 or not 1 <= val <= 8:
                raise NotDecoded(UNSUPPORTED, "orientation tag not a SHORT 1..8")
            return val
    return 1


def parse(data):
    """Marker walk.  -> dict; raises NotDecoded(status, why)."""
    d = bytes(data)
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise NotDecoded(MALFORMED, "no SOI")
    p = 2
    qt = [None] * 4
    dht = {}  # (class, id) -> (counts, symbols)
    dri = 0
    sof = None
    jfif = adobe = False
    adobe_transform = 0
    orientation = None
    while True:
        if p + 2 > n or d[p] != 0xFF:
            raise NotDecoded(MALFORMED, "marker expected at %d" % p)
        while p + 1 < n and d[p + 1] == 0xFF:  # fill bytes
            p += 1
        if p + 2 > n:
            raise NotDecoded(MALFORMED, "truncated marker")
        m = d[p + 1]
        p += 2
        if m == 0xD8 or m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise NotDecoded(MALFORMED, "marker %02X out of place" % m)
        if p + 2 > n:
            raise NotDecoded(MALFORMED, "truncated length")
        L = _u16(d, p)
        if L < 2 or p + L > n:
            raise NotDecoded(MALFORMED, "segment length")
        s = d[p + 2:p + L]
        p += L
        if m == 0xDB:  # DQT
            i = 0
            while i < len(s):
                pq, tq = s[i] >> 4, s[i] & 15
                if pq > 1 or tq > 3 or i + 1 + 64 * (pq + 1) > len(s):
                    raise NotDecoded(MALFORMED, "DQT")
                if pq == 0:
                    v = np.frombuffer(s, np.uint8, 64, i + 1).astype(np.int64)
                else:
                    v = np.frombuffer(s, ">u2", 64, i + 1).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = v
                qt[tq] = q
                i += 1 + 64 * (pq + 1)
        elif m == 0xC4:  # DHT
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
        elif m == 0xDD:  # DRI
            if len(s) != 2:
                raise NotDecoded(MALFORMED, "DRI")
            dri = _u16(s, 0)
        elif m in (0xC0, 0xC1):
            if sof is not None or len(s) < 6:
                raise NotDecoded(MALFORMED, "SOF")
            prec, hh, ww, nf = s[0], _u16(s, 1), _u16(s, 3), s[5]
            if len(s) != 6 + 3 * nf:
                raise NotDecoded(MALFORMED, "SOF length")
            if prec != 8:
                raise NotDecoded(UNSUPPORTED, "%d-bit samples" % prec)
            if hh == 0 or ww == 0:
                raise NotDecoded(UNSUPPORTED, "zero / DNL height")
            if nf not in (1, 3):
                raise NotDecoded(UNSUPPORTED, "%d components" % nf)
            comps = [(s[6 + 3 * c], s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]) for c in range(nf)]
            if len(set(c[0] for c in comps)) != nf or any(c[3] > 3 for c in comps):
                raise NotDecoded(MALFORMED, "component ids / table ids")
            if nf == 1:
                comps = [(comps[0][0], 1, 1, comps[0][3])]  # one component: one block per MCU whatever its factors say
            elif not (comps[0][1] in (1, 2) and comps[0][2] in (1, 2) and all(c[1] == 1 and c[2] == 1 for c in comps[1:])):
                raise NotDecoded(UNSUPPORTED, "sampling factors")
            sof = (hh, ww, comps)
        elif 0xC2 <= m <= 0xCF:
            raise NotDecoded(UNSUPPORTED, "SOF%d / DAC / JPG" % (m - 0xC0))
        elif m == 0xE0:
            if len(s) >= 14 and s[:5] == b"JFIF\x00":
                jfif = True
        elif m == 0xEE:
            if len(s) >= 12 and s[:5] == b"Adobe":
                adobe, adobe_transform = True, s[11]
        elif m == 0xE1:
            o = _exif_orientation(s)
            if o is not None:
                if orientation is not None:
                    raise NotDecoded(UNSUPPORTED, "two EXIF blocks")
                orientation = o
        elif 0xE2 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            break
        else:
            raise NotDecoded(UNSUPPORTED, "marker %02X" % m)
    # SOS
    if sof is None:
        raise NotDecoded(MALFORMED, "SOS before SOF")
    hh, ww, comps = sof
    nf = len(comps)
    if len(s) < 1 or s[0] != nf or len(s) != 4 + 2 * nf:
        raise NotDecoded(UNSUPPORTED, "scan is not one interleaved scan of every component")
    tabs = []
    for c in range(nf):
        if s[1 + 2 * c] != comps[c][0]:
            raise NotDecoded(UNSUPPORTED, "scan component order")
        td, ta = s[2 + 2 * c] >> 4, s[2 + 2 * c] & 15
        if (0, td) not in dht or (1, ta) not in dht or qt[comps[c][3]] is None:
            raise NotDecoded(UNSUPPORTED, "table not defined")
        if any(v > 15 for v in dht[(0, td)][1]):
            raise NotDecoded(MALFORMED, "DC symbol > 15")
        if any(v > 32767 for v in qt[comps[c][3]]):
            raise NotDecoded(UNSUPPORTED, "quantiser above 32767")
        tabs.append((td, ta))
    for td, ta in tabs:
        _check_canonical(dht[(0, td)][0])
        _check_canonical(dht[(1, ta)][0])
    if tuple(s[1 + 2 * nf:4 + 2 * nf]) != (0, 63, 0):
        raise NotDecoded(UNSUPPORTED, "Ss/Se/Ah/Al of a sequential scan")
    if nf == 3:
        if jfif:
            ycc = True
        elif adobe:
            ycc = adobe_transform != 0
        else:
            ycc = tuple(c[0] for c in comps) != (82, 71, 66)
        if not ycc:
            raise NotDecoded(UNSUPPORTED, "RGB colour space")
    if hh * ww > MAX_PIXELS:
        raise NotDecoded(TOO_LARGE, "over the pixel cap")
    hmax, vmax = comps[0][1], comps[0][2]
    mcux, mcuy = -(-ww // (8 * hmax)), -(-hh // (8 * vmax))
    nmcu = mcux * mcuy
    nseg = -(-nmcu // dri) if dri else 1
    # entropy-coded data: FF 00 is a stuffed FF, FF D0..D7 a restart marker, FF D9 the end; anything else is not decoded
    segs = []
    start, q = p, p
    while True:
        q = d.find(b"\xff", q)
        if q < 0 or q + 1 >= n:
            raise NotDecoded(MALFORMED, "no EOI")
        m = d[q + 1]
        if m == 0:
            q += 2
            continue
        if 0xD0 <= m <= 0xD7:
            if not dri or m - 0xD0 != len(segs) % 8:
                raise NotDecoded(CORRUPT, "restart marker out of sequence")
            segs.append((start, q))
            start = q = q + 2
            continue
        if m != 0xD9:
            raise NotDecoded(UNSUPPORTED, "marker %02X after the scan" % m)
        segs.append((start, q))
        break
    if len(segs) != nseg:
        raise NotDecoded(CORRUPT, "%d restart segments, %d expected" % (len(segs), nseg))
    H, W = (ww, hh) if orientation and orientation >= 5 else (hh, ww)
    return dict(h=hh, w=ww, out_h=H, out_w=W, orientation=orientation or 1, comps=comps, hmax=hmax, vmax=vmax, mcux=mcux,
                mcuy=mcuy, nmcu=nmcu, dri=dri, segments=segs, qt=[qt[c[3]] for c in comps],
                dc=[dht[(0, t[0])] for t in tabs], ac=[dht[(1, t[1])] for t in tabs])


def info(data):
    """-> (status, out_h, out_w, orientation): what smapb_jpeg_info reports (header-level acceptance only)."""
    try:
        hd = parse(data)
    except NotDecoded as e:
        return e.status, 0, 0, 0
    return OK, hd["out_h"], hd["out_w"], hd["orientation"]


def _unstuff(d):
    return d.replace(b"\xff\x00", b"\xff")


def mcu_layout(hd):
    """Component index of each block of an MCU, in decode order."""
    lay = []
    for c, comp in enumerate(hd["comps"]):
        lay += [c] * (comp[1] * comp[2])
    return lay


def entropy_decode(data, hd):
    """-> int16 [nmcu * blocks_per_mcu, 64] in natural order with absolute DC, in decode order (MCU by MCU).  A code that is not
    in its table, a run past coefficient 63 or data that ends before the segment's last MCU raise NotDecoded(CORRUPT); bits
    left over after a segment's last MCU are ignored."""
    d = bytes(data)
    lay = mcu_layout(hd)
    bpm = len(lay)
    dcl = [_huff_table(*t) for t in hd["dc"]]
    acl = [_huff_table(*t) for t in hd["ac"]]
    out = np.zeros((hd["nmcu"] * bpm, 64), np.int16)
    per = hd["dri"] or hd["nmcu"]
    zz = ZIGZAG.tolist()
    for si, (a, b) in enumerate(hd["segments"]):
        buf = _unstuff(d[a:b])
        nbits = len(buf) * 8
        buf += b"\x00" * 8
        m0 = si * per
        m1 = min(hd["nmcu"], m0 + per)
        pred = [0] * len(hd["comps"])
        pos = 0

        def unit(lut):  # one code and its extra bits -> (symbol, value, new pos)
            i = pos >> 3
            w = int.from_bytes(buf[i:i + 5], "big") << (pos & 7)
            e = lut[(w >> 24) & 0xFFFF]
            if e == 0:
                raise NotDecoded(CORRUPT, "code not in table")
            ln, sym = e >> 8, e & 255
            s = sym & 15
            v = 0
            if s:
                v = (w >> (40 - ln - s)) & ((1 << s) - 1)
                if v < (1 << (s - 1)):
                    v += 1 - (1 << s)
            if pos + ln + s > nbits:
                raise NotDecoded(CORRUPT, "data exhausted")
            return sym, v, pos + ln + s

        for mcu in range(m0, m1):
            for j, c in enumerate(lay):
                blk = out[mcu * bpm + j]
                sym, v, pos = unit(dcl[c])
                pred[c] += v
                blk[0] = np.int16(((pred[c] + 32768) & 0xFFFF) - 32768)
                k = 1
                while k < 64:
                    sym, v, pos = unit(acl[c])
                    r, s = sym >> 4, sym & 15
                    if s == 0:
                        if r != 15:
                            break
                        k += 16
                        if k > 64:
                            raise NotDecoded(CORRUPT, "run past coefficient 63")
                        continue
                    k += r
                    if k > 63:
                        raise NotDecoded(CORRUPT, "run past coefficient 63")
                    blk[zz[k]] = v
                    k += 1
    return out


# accurate-integer IDCT constants: round(c * 2^13)
C0_298, C0_390, C0_541, C0_765, C0_899, C1_175, C1_501, C1_847 = 2446, 3196, 4433, 6270, 7373, 9633, 12299, 15137
C1_961, C2_053, C2_562, C3_072 = 16069, 16819, 20995, 25172


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, shift):
    """LL&M 8-point IDCT on int64 arrays; outputs (sum + 2^(shift-1)) >> shift."""
    z1 = (x2 + x6) * C0_541
    t2 = z1 - x6 * C1_847
    t3 = z1 + x2 * C0_765
    t0 = (x0 + x4) << 13
    t1 = (x0 - x4) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    a0, a1, a2, a3 = x7, x5, x3, x1
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * C1_175
    a0, a1, a2, a3 = a0 * C0_298, a1 * C2_053, a2 * C3_072, a3 * C1_501
    z1, z2, z3, z4 = z1 * -C0_899, z2 * -C2_562, z3 * -C1_961 + z5, z4 * -C0_390 + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    r = 1 << (shift - 1)
    return [(t10 + a3 + r) >> shift, (t11 + a2 + r) >> shift, (t12 + a1 + r) >> shift, (t13 + a0 + r) >> shift,
            (t13 - a0 + r) >> shift, (t12 - a1 + r) >> shift, (t11 - a2 + r) >> shift, (t10 - a3 + r) >> shift]


def idct_blocks(coef, q):
    """coef int16 [N,64] natural order, q int [64] -> uint8 [N,8,8].  Pass 1 (columns) keeps 2 extra bits
    ((x << 13) >> 11), pass 2 (rows) removes 13 + 2 + 3 bits, then + 128 and range limiting."""
    c = coef.astype(np.int64).reshape(-1, 8, 8) * np.asarray(q, np.int64).reshape(8, 8)
    cols = _idct_1d(*[c[:, k, :] for k in range(8)], 11)  # each [N, 8 cols]
    ws = np.stack(cols, axis=1)                                    # [N, 8 rows, 8 cols]
    if np.abs(c).max(initial=0) > GUARD or np.abs(ws).max(initial=0) > GUARD:
        raise NotDecoded(UNSUPPORTED, "IDCT operands beyond the 16-bit range of cv2's SIMD IDCT")
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)], 18)
    v = np.stack(rows, axis=2)
    if IDCT_CLAMP:
        return np.clip(v + 128, 0, 255).astype(np.uint8)
    u = v & 0x3FF
    u = np.where(u >= 512, u - 1024, u)
    return np.clip(u + 128, 0, 255).astype(np.uint8)


def idct_planes(coef, hd):
    """-> list of uint8 planes, one per component, padded to whole MCUs."""
    lay = mcu_layout(hd)
    bpm = len(lay)
    mx, my = hd["mcux"], hd["mcuy"]
    planes = []
    j0 = 0
    for c, (cid, hs, vs, tq) in enumerate(hd["comps"]):
        idx = (np.arange(hd["nmcu"])[:, None] * bpm + j0 + np.arange(hs * vs)[None, :]).reshape(-1)
        px = idct_blocks(coef[idx], hd["qt"][c])  # [nmcu*hs*vs, 8, 8]
        px = px.reshape(my, mx, vs, hs, 8, 8).transpose(0, 2, 4, 1, 3, 5).reshape(my * vs * 8, mx * hs * 8)
        planes.append(px)
        j0 += hs * vs
    return planes


def upsample(C, hs, vs, H, W, hmax, vmax):
    """Chroma plane (padded) at factors (1,1) -> full-resolution int plane [H, W] (libjpeg's fancy upsampling)."""
    cw, ch = -(-W // hmax), -(-H // vmax)
    C = C[:ch, :cw].astype(np.int64)
    if hmax == 1 and vmax == 1:
        return C
    if hmax == 2 and cw <= 2 and vmax in (1, 2):  # libjpeg's fancy h2 filters need 3 columns: plain replication
        out = np.repeat(C, 2, axis=1)
        if vmax == 2:
            out = np.repeat(out, 2, axis=0)
        return out[:H, :W]
    if vmax == 2:
        up = np.concatenate([C[:1], C[:-1]], 0)
        dn = np.concatenate([C[1:], C[-1:]], 0)
        if hmax == 1:
            out = np.empty((2 * ch, cw), np.int64)
            out[0::2] = (3 * C + up + 1) >> 2
            out[1::2] = (3 * C + dn + 2) >> 2
            return out[:H, :W]
        rows = np.empty((2 * ch, cw), np.int64)  # column sums of the nearer and the further row
        rows[0::2] = 3 * C + up
        rows[1::2] = 3 * C + dn
        b_even, b_odd, sh = 8, 7, 4
    else:
        rows = C
        b_even, b_odd, sh = 1, 2, 2
    lf = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    rt = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((rows.shape[0], 2 * cw), np.int64)
    out[:, 0::2] = (3 * rows + lf + b_even) >> sh
    out[:, 1::2] = (3 * rows + rt + b_odd) >> sh
    return out[:H, :W]


def orient(img, o):
    """EXIF orientation as cv2 applies it: 2 flip x, 3 rotate 180, 4 flip y, 5 transpose, 6 rotate 90 clockwise,
    7 transverse, 8 rotate 90 counter-clockwise."""
    if o in (5, 6, 7, 8):
        img = img.transpose(1, 0, 2)
        o = {5: 1, 6: 2, 7: 3, 8: 4}[o]
    if o == 2:
        img = img[:, ::-1]
    elif o == 3:
        img = img[::-1, ::-1]
    elif o == 4:
        img = img[::-1]
    return np.ascontiguousarray(img)


def colour(planes, hd):
    H, W = hd["h"], hd["w"]
    Y = planes[0][:H, :W].astype(np.int64)
    if len(planes) == 1:
        bgr = np.repeat(Y[:, :, None], 3, axis=2).astype(np.uint8)
    else:
        cb = upsample(planes[1], 1, 1, H, W, hd["hmax"], hd["vmax"]) - 128
        cr = upsample(planes[2], 1, 1, H, W, hd["hmax"], hd["vmax"]) - 128
        half = 1 << 15
        r = Y + ((91881 * cr + half) >> 16)
        g = Y + ((-46802 * cr - 22554 * cb + half) >> 16)
        b = Y + ((116130 * cb + half) >> 16)
        bgr = np.clip(np.stack([b, g, r], 2), 0, 255).astype(np.uint8)
    return orient(bgr, hd["orientation"])


def decode(data):
    """-> uint8 BGR [H, W, 3] as cv2.imread(path, IMREAD_COLOR) returns it; NotDecoded for inputs the GPU decoder leaves to cv2."""
    hd = parse(data)
    return colour(idct_planes(entropy_decode(data, hd), hd), hd)
