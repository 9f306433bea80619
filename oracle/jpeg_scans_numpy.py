"""CPU restatement of the multi-scan JPEG decoding of smap_b200/csrc/jpeg.cu (SMAPB_JPEG_SCANS): sequential files with
several scans and progressive Huffman files (ITU-T T.81 Annex G: DC first and refinement, AC first with EOB runs, AC
refinement, non-interleaved scans on the component's own block grid).  The IDCT, upsampling, colour conversion and
orientation are jpeg_numpy's; so is the coefficient layout (frame MCU by frame MCU) that feeds them.

    hd = parse(data)                  # every scan up to EOI, jpeg_parse's rules with SMAPB_JPEG_SCANS; NotDecoded otherwise
    coef = entropy_decode(data, hd)   # int16 [nmcu * blocks_per_mcu, 64] after every scan
    decode(data)                      # -> uint8 BGR as cv2.imread returns it
"""
import numpy as np

from . import jpeg_numpy as J
from .jpeg_numpy import CORRUPT, MALFORMED, OK, TOO_LARGE, UNSUPPORTED, NotDecoded

MAX_SCANS = 64
MAX_SCAN_BYTES = 1 << 28
# libjpeg-turbo 3.x (cv2's bundled build) smooths progressive output (block smoothing) when a coefficient of zig-zag index
# 1..SAVED_COEFS-1 of a component is not fully refined; such files are not decoded (a test lowers it to 1 to get the plain
# IDCT result and show that cv2's differs)
SAVED_COEFS = 10


def parse(data):
    d = bytes(data)
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise NotDecoded(MALFORMED, "no SOI")
    p = 2
    qt = [None] * 4
    qt_used = [False] * 4
    dht = {}
    dri = 0
    sof = None
    progressive = False
    jfif = adobe = False
    adobe_transform = 0
    orientation = None
    latched = {}
    coef_bits = None
    nscanned = None
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
                v = np.frombuffer(s, np.uint8 if pq == 0 else ">u2", 64, i + 1).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[J.ZIGZAG] = v
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
            if prec != 8 or hh == 0 or ww == 0 or nf not in (1, 3):
                raise NotDecoded(UNSUPPORTED, "precision / size / components")
            comps = [(s[6 + 3 * c], s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]) for c in range(nf)]
            for c in range(nf):
                if comps[c][3] > 3 or any(comps[e][0] == comps[c][0] for e in range(c)):
                    raise NotDecoded(MALFORMED, "component ids / table ids")
            if nf == 1:
                comps = [(comps[0][0], 1, 1, comps[0][3])]
            elif not (comps[0][1] in (1, 2) and comps[0][2] in (1, 2) and all(c[1] == 1 and c[2] == 1 for c in comps[1:])):
                raise NotDecoded(UNSUPPORTED, "sampling factors")
            if hh * ww > J.MAX_PIXELS:
                raise NotDecoded(TOO_LARGE, "over the pixel cap")
            hmax, vmax = comps[0][1], comps[0][2]
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
            if len(scans) == MAX_SCANS:
                raise NotDecoded(UNSUPPORTED, "more than %d scans" % MAX_SCANS)
            hh, ww, comps = sof
            nf = len(comps)
            ns = s[0] if len(s) >= 1 else 0
            if ns < 1 or ns > nf or len(s) != 4 + 2 * ns:
                raise NotDecoded(MALFORMED, "SOS length")
            ss, se, ah, al = s[1 + 2 * ns], s[2 + 2 * ns], s[3 + 2 * ns] >> 4, s[3 + 2 * ns] & 15
            sc = []
            for k in range(ns):
                ids = [c[0] for c in comps]
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
                dc_band = ss == 0
                if (se != 0) if dc_band else (ss > se or se > 63 or ns != 1):
                    raise NotDecoded(UNSUPPORTED, "bad spectral selection")
                if (ah != 0 and al != ah - 1) or al > 13:
                    raise NotDecoded(UNSUPPORTED, "bad successive approximation")
                for c in sc:
                    cb = coef_bits[c]
                    if not dc_band and cb[0] < 0:
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
            if segs[-1][1] - segs[0][0] > MAX_SCAN_BYTES:
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
        if any(b != 0 for b in coef_bits[c][1:SAVED_COEFS]):
            raise NotDecoded(UNSUPPORTED, "coefficient 1..9 not fully refined: libjpeg-turbo smooths the output")
    if nf == 3:
        if jfif:
            ycc = True
        elif adobe:
            ycc = adobe_transform != 0
        else:
            ycc = tuple(c[0] for c in comps) != (82, 71, 66)
        if not ycc:
            raise NotDecoded(UNSUPPORTED, "RGB colour space")
    H, W = (ww, hh) if orientation and orientation >= 5 else (hh, ww)
    return dict(h=hh, w=ww, out_h=H, out_w=W, orientation=orientation or 1, comps=comps, hmax=hmax, vmax=vmax, mcux=mcux,
                mcuy=mcuy, nmcu=mcux * mcuy, qt=[latched[c] for c in range(nf)], scans=scans, progressive=progressive)


def info(data):
    """-> (status, out_h, out_w, orientation): what smapb_jpeg_info_ex(SMAPB_JPEG_SCANS) reports."""
    try:
        hd = parse(data)
    except NotDecoded as e:
        return e.status, 0, 0, 0
    return OK, hd["out_h"], hd["out_w"], hd["orientation"]


def _block_index(hd, sc, b):
    """Scan block b (decode order) -> block of the coefficient buffer (frame MCU by frame MCU)."""
    comps = hd["comps"]
    bpm = sum(c[1] * c[2] for c in comps)
    j0 = [sum(comps[e][1] * comps[e][2] for e in range(c)) for c in range(len(comps))]
    if len(sc["comps"]) > 1:
        m, j = divmod(b, sc["bpm"])
        for c in sc["comps"]:
            nb = comps[c][1] * comps[c][2]
            if j < nb:
                return m * bpm + j0[c] + j
            j -= nb
    c = sc["comps"][0]
    h, v = comps[c][1], comps[c][2]
    by, bx = divmod(b, sc["mcux"])
    return ((by // v) * hd["mcux"] + bx // h) * bpm + j0[c] + (by % v) * h + bx % h


class _Bits:
    def __init__(self, buf):
        self.buf = buf + b"\x00" * 8
        self.n = len(buf) * 8
        self.pos = 0

    def get(self, k):
        if self.pos + k > self.n:
            raise NotDecoded(CORRUPT, "data exhausted")
        i = self.pos >> 3
        w = int.from_bytes(self.buf[i:i + 5], "big") << (self.pos & 7)
        self.pos += k
        return (w >> (40 - k)) & ((1 << k) - 1) if k else 0

    def huff(self, lut):
        i = self.pos >> 3
        w = int.from_bytes(self.buf[i:i + 5], "big") << (self.pos & 7)
        e = lut[(w >> 24) & 0xFFFF]
        if e == 0:
            raise NotDecoded(CORRUPT, "code not in table")
        if self.pos + (e >> 8) > self.n:
            raise NotDecoded(CORRUPT, "data exhausted")
        self.pos += e >> 8
        return e & 255


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(data, hd):
    """-> int16 [nmcu * blocks_per_mcu, 64], natural order, after every scan.  Errors (a code not in its table, a run past
    Se, a correction symbol other than 1, data that ends before a segment's last block) raise NotDecoded(CORRUPT)."""
    d = bytes(data)
    comps = hd["comps"]
    bpm = sum(c[1] * c[2] for c in comps)
    coef = np.zeros((hd["nmcu"] * bpm, 64), np.int64)
    zz = J.ZIGZAG.tolist()
    for sc in hd["scans"]:
        ss, se, ah, al = sc["ss"], sc["se"], sc["ah"], sc["al"]
        dcl = [J._huff_table(*t) if t else None for t in sc["dc"]]
        acl = [J._huff_table(*t) if t else None for t in sc["ac"]]
        lay = []
        for k, c in enumerate(sc["comps"]):
            lay += [k] * (comps[c][1] * comps[c][2] if len(sc["comps"]) > 1 else 1)
        per = sc["dri"] or sc["nmcu"]
        p1, m1 = 1 << al, -(1 << al)
        for si, (a, b) in enumerate(sc["segments"]):
            bits = _Bits(J._unstuff(d[a:b]))
            pred = [0] * len(lay)
            eobrun = 0
            for mcu in range(si * per, min(sc["nmcu"], (si + 1) * per)):
                for j, k in enumerate(lay):
                    blk = coef[_block_index(hd, sc, mcu * sc["bpm"] + j)]
                    if ss == 0 and ah == 0:  # sequential or DC first
                        s = bits.huff(dcl[k])
                        pred[k] += _extend(bits.get(s), s)
                        blk[0] = ((((pred[k] << al) & 0xFFFF) + 32768) & 0xFFFF) - 32768
                        if se == 0:
                            continue
                    if ss == 0 and ah > 0:  # DC refinement
                        if bits.get(1):
                            blk[0] |= p1
                        continue
                    if ah == 0:  # sequential AC, AC first
                        if eobrun:
                            eobrun -= 1
                            continue
                        i = max(ss, 1)
                        while i <= se:
                            sym = bits.huff(acl[k])
                            r, s = sym >> 4, sym & 15
                            if s == 0:
                                if r == 15:
                                    i += 16
                                    if i > se + 1:
                                        raise NotDecoded(CORRUPT, "run past Se")
                                    continue
                                if ss > 0:
                                    eobrun = (1 << r) + bits.get(r) - 1
                                break
                            i += r
                            if i > se:
                                raise NotDecoded(CORRUPT, "run past Se")
                            blk[zz[i]] = ((((_extend(bits.get(s), s) << al) & 0xFFFF) + 32768) & 0xFFFF) - 32768
                            i += 1
                        continue
                    # AC refinement
                    i = ss
                    if eobrun == 0:
                        while i <= se:
                            sym = bits.huff(acl[k])
                            r, s = sym >> 4, sym & 15
                            sv = 0
                            if s:
                                if s != 1:
                                    raise NotDecoded(CORRUPT, "refinement symbol with size != 1")
                                sv = p1 if bits.get(1) else m1
                            elif r != 15:
                                eobrun = (1 << r) + bits.get(r)
                                break
                            while i <= se:
                                z = zz[i]
                                if blk[z] != 0:
                                    if bits.get(1) and (blk[z] & p1) == 0:
                                        blk[z] += p1 if blk[z] >= 0 else m1
                                else:
                                    r -= 1
                                    if r < 0:
                                        break
                                i += 1
                            if sv:
                                if i > se:
                                    raise NotDecoded(CORRUPT, "run past Se")
                                blk[zz[i]] = sv
                            i += 1
                    if eobrun > 0:
                        while i <= se:
                            z = zz[i]
                            if blk[z] != 0 and bits.get(1) and (blk[z] & p1) == 0:
                                blk[z] += p1 if blk[z] >= 0 else m1
                            i += 1
                        eobrun -= 1
    return coef.astype(np.int16)


def decode(data):
    """-> uint8 BGR [H, W, 3] as cv2.imread(path, IMREAD_COLOR) returns it; NotDecoded for inputs left to cv2."""
    hd = parse(data)
    return J.colour(J.idct_planes(entropy_decode(data, hd), hd), hd)
