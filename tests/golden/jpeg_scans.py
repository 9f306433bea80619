"""Seeded multi-scan JPEG corpus for the GPU decoder's SMAPB_JPEG_SCANS path (tests/test_jpeg_scans_cpu.py,
tests/test_jpeg_scans_gpu.py), written by cv2 and Pillow at test time: progressive files in the four samplings and in
grayscale, with restart intervals, optimised tables and EXIF orientations, and damaged progressive files."""
import io

import numpy as np

from jpeg_corpus import SAMPLINGS, SMALL, content, cv2_jpeg, exif_block


def cv2_progressive(img, q=90, samp="420", rst=0):
    import cv2

    p = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[samp]]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    ok, b = cv2.imencode(".jpg", img, p)
    assert ok
    b = b.tobytes()
    assert not rst or b"\xff\xdd" in b[:scan_header_end(b)]  # the file carries its DRI
    return b


def pil_progressive(img_bgr, q=90, subsampling=2, orientation=None, gray=False, **kw):
    from PIL import Image

    bio = io.BytesIO()
    args = dict(quality=q, progressive=True, **kw)
    if not gray:
        args["subsampling"] = subsampling
    if orientation is not None:
        args["exif"] = exif_block(orientation)
    im = Image.fromarray(np.ascontiguousarray(img_bgr[:, :, 1] if gray else img_bgr[:, :, ::-1]))
    im.save(bio, "JPEG", **args)
    return bio.getvalue()


def scan_header_end(b):
    """Offset just past the first SOS header."""
    p = 2
    while True:
        m, L = b[p + 1], (b[p + 2] << 8) | b[p + 3]
        p += 2 + L
        if m == 0xDA:
            return p


def sos_offsets(b):
    """Offsets of every SOS marker."""
    out, i = [], b.find(b"\xff\xda")
    while i >= 0:
        out.append(i)
        i = b.find(b"\xff\xda", i + 2)
    return out


def corpus(large=False, seed=15):
    """-> list of (name, bytes) SMAPB_JPEG_SCANS decodes.  large=True adds 832x512 and 1920x1080 frames."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in SMALL:
        for kind in ("flat", "noise", "check"):
            img = content(kind, h, w, rng)
            for q in (50, 95):
                for s in SAMPLINGS:
                    out.append(("prog_%dx%d_%s_q%d_%s" % (w, h, kind, q, s), cv2_progressive(img, q, s)))
                out.append(("prog_%dx%d_%s_q%d_gray" % (w, h, kind, q), cv2_progressive(img[:, :, 1].copy(), q)))
            out.append(("pil_%dx%d_%s" % (w, h, kind), pil_progressive(img, 90)))
            out.append(("pil_%dx%d_%s_gray" % (w, h, kind), pil_progressive(img, 90, gray=True)))
    img = content("noise", 37, 61, rng)
    for rst in (1, 7):
        for s in SAMPLINGS:
            out.append(("prog_rst%d_%s" % (rst, s), cv2_progressive(img, 90, s, rst=rst)))
    out.append(("prog_rst3_gray", cv2_progressive(img[:, :, 0].copy(), 90, rst=3)))
    for sub in (0, 1, 2):
        out.append(("pil_opt_sub%d" % sub, pil_progressive(img, 85, sub, optimize=True)))
    out.append(("pil_opt_gray", pil_progressive(img, 85, gray=True, optimize=True)))
    img2 = content("smooth", 40, 64, rng)
    for o in range(1, 9):
        out.append(("pil_exif%d" % o, pil_progressive(img2, 90, 2, o)))
    out.append(("baseline_420", cv2_jpeg(img, 90, "420")))  # single-scan files take the same path
    out.append(("baseline_gray_rst", cv2_jpeg(img[:, :, 0].copy(), 90, rst=5)))
    if large:
        for h, w in ((512, 832), (1080, 1920)):
            big = content("smooth", h, w, rng)
            for s in SAMPLINGS:
                out.append(("prog_%dx%d_q90_%s" % (w, h, s), cv2_progressive(big, 90, s)))
            out.append(("prog_%dx%d_rst5_420" % (w, h), cv2_progressive(big, 90, "420", rst=5)))
            out.append(("pil_%dx%d_opt" % (w, h), pil_progressive(big, 90, 2, optimize=True)))
            out.append(("pil_%dx%d_gray" % (w, h), pil_progressive(big, 90, gray=True)))
    return out


def large_frames(seed=19):
    """4032x3024 progressive frames written by cv2 (4:2:0 smooth, 4:4:4 noise) and 1920x1080 noise."""
    rng = np.random.default_rng(seed)
    return [("prog_1920x1080_noise_q95_420", cv2_progressive(content("noise", 1080, 1920, rng), 95, "420")),
            ("prog_4032x3024_smooth_q90_420", cv2_progressive(content("smooth", 3024, 4032, rng), 90, "420")),
            ("prog_4032x3024_noise_q90_444", cv2_progressive(content("noise", 3024, 4032, rng), 90, "444"))]


def damaged(seed=17):
    """Damaged progressive files: cuts at and inside every scan, flipped bytes in the later (refinement) scans, a wrong
    restart marker."""
    rng = np.random.default_rng(seed)
    img = content("noise", 37, 61, rng)
    base = [cv2_progressive(img, 90, "420"), cv2_progressive(img, 75, "444", rst=3),
            pil_progressive(content("smooth", 64, 96, rng), 90, 1, optimize=True)]
    out = []
    for k, b in enumerate(base):
        sos = sos_offsets(b)
        for j, s in enumerate(sos):
            out.append(("cut%d_at_scan%d" % (k, j), b[:s]))
            nxt = sos[j + 1] if j + 1 < len(sos) else len(b) - 2
            out.append(("cut%d_in_scan%d" % (k, j), b[:(s + nxt) // 2]))
        for j, pos in enumerate(rng.integers(sos[len(sos) // 2], len(b) - 2, 8)):
            c = bytearray(b)
            c[pos] ^= int(rng.integers(1, 256))
            out.append(("flip%d_%d" % (k, j), bytes(c)))
    b = base[1]
    i = b.find(b"\xff\xd1", scan_header_end(b))
    c = bytearray(b)
    c[i + 1] = 0xD5
    out.append(("rst_out_of_sequence", bytes(c)))
    return out


# ---- lossless transcoder -----------------------------------------------------------------------------------------------
# Rewrites the quantised coefficients of a baseline file (oracle/jpeg_numpy.py's entropy_decode) with any scan script, as
# libjpeg's encoder codes each scan type (jcphuff.c's rules: point transforms, EOB runs up to 32767, correction bits held
# back while an EOB run is open), with per-scan optimised Huffman tables and optional restart intervals.  A script is a
# list of (components, Ss, Se, Ah, Al); component indices are the frame's.  Nothing here depends on the GPU decoder:
# for a complete script cv2.imread(transcoded) equals cv2.imread(original).

ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35,
      42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]

# libjpeg's jpeg_simple_progression for YCbCr (what cv2 writes with IMWRITE_JPEG_PROGRESSIVE)
SCRIPT_LIBJPEG = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((0,), 6, 63, 0, 2),
                  ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
SCRIPTS = {
    # sequential (SOF0) with several scans
    "seq_per_component": [((0,), 0, 63, 0, 0), ((1,), 0, 63, 0, 0), ((2,), 0, 63, 0, 0)],
    "seq_luma_then_chroma": [((0,), 0, 63, 0, 0), ((1, 2), 0, 63, 0, 0)],
    # progressive (SOF2)
    "libjpeg": SCRIPT_LIBJPEG,
    "mozjpeg_like": [((0,), 0, 0, 0, 0), ((1,), 0, 0, 0, 0), ((2,), 0, 0, 0, 0), ((0,), 1, 2, 0, 0), ((0,), 3, 63, 0, 0),
                     ((1,), 1, 9, 0, 0), ((2,), 1, 9, 0, 0), ((1,), 10, 63, 0, 0), ((2,), 10, 63, 0, 0)],
    "spectral_only": [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 1, 0, 0), ((0,), 2, 9, 0, 0), ((0,), 10, 63, 0, 0),
                      ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)],
    "approximation_deep": [((0,), 0, 0, 0, 3), ((1,), 0, 0, 0, 2), ((2,), 0, 0, 0, 2), ((0,), 1, 63, 0, 3),
                           ((1, 2), 0, 0, 2, 1), ((0,), 0, 0, 3, 2), ((0,), 1, 63, 3, 2), ((1,), 1, 63, 0, 1),
                           ((0,), 0, 0, 2, 1), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0), ((1, 2), 0, 0, 1, 0),
                           ((2,), 1, 63, 0, 0), ((0,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0)],
}
SEQUENTIAL = ("seq_per_component", "seq_luma_then_chroma")


def for_components(script, nf):
    """The script restricted to components < nf (a grayscale file keeps the luma scans)."""
    out = []
    for comps, ss, se, ah, al in script:
        c = tuple(x for x in comps if x < nf)
        if c:
            out.append((c, ss, se, ah, al))
    return out


def _optimal_table(freq):
    """libjpeg's jpeg_gen_optimal_table: code lengths <= 16 from symbol counts -> (counts[16], symbols)."""
    freq = list(freq) + [1]  # symbol 256 reserves the all-ones code
    n = len(freq)
    codesize, others = [0] * n, [-1] * n
    f = list(freq)
    while True:
        c1 = c2 = -1
        v1 = v2 = None
        for i in range(n):
            if f[i] and (v1 is None or f[i] <= v1):
                v1, c1 = f[i], i
        for i in range(n):
            if f[i] and i != c1 and (v2 is None or f[i] <= v2):
                v2, c2 = f[i], i
        if c2 < 0:
            break
        f[c1] += f[c2]
        f[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for i in range(n):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1  # drop the reserved code
    syms = [s for size in range(1, 33) for s in range(256) if codesize[s] == size]
    return bits[1:17], syms


def _codes(counts, syms):
    code, k, out = 0, 0, {}
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            out[syms[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


class _Writer:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def bits(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self):
        if self.n:
            self.bits(0x7F, 8 - self.n)


def _nbits(v):
    return int(abs(int(v))).bit_length()


def _scan_tokens(coef, hd, comps, ss, se, ah, al, dri):
    """Symbols and raw bits of one scan: a list of ('s', table key, symbol) / ('b', value, n) / ('rst',)."""
    from oracle import jpeg_scans_numpy as S

    fc = hd["comps"]
    inter = len(comps) > 1
    if inter:
        mcux, nmcu = hd["mcux"], hd["nmcu"]
        lay = [(k, j) for k, c in enumerate(comps) for j in range(fc[c][1] * fc[c][2])]
    else:
        c = comps[0]
        cw, ch = -(-hd["w"] * fc[c][1] // hd["hmax"]), -(-hd["h"] * fc[c][2] // hd["vmax"])
        mcux = -(-cw // 8)
        nmcu = mcux * -(-ch // 8)
        lay = [(0, 0)]
    sc = dict(comps=list(comps), bpm=len(lay), mcux=mcux)
    toks = []
    pred = [0] * len(comps)
    eob = [0, []]  # EOBRUN, correction bits held back (BE)

    def emit_eobrun(k):
        if eob[0]:
            n = eob[0].bit_length() - 1
            toks.append(("s", ("ac", k), n << 4))
            if n:
                toks.append(("b", eob[0] & ((1 << n) - 1), n))
            for b in eob[1]:
                toks.append(("b", b, 1))
            eob[0], eob[1] = 0, []

    for m in range(nmcu):
        if dri and m and m % dri == 0:
            emit_eobrun(0)
            toks.append(("rst",))
            pred = [0] * len(comps)
        for j, (k, _) in enumerate(lay):
            blk = coef[S._block_index(hd, sc, m * len(lay) + j)].astype(np.int64)
            if ss == 0:
                if ah == 0:
                    v = int(blk[0]) >> al
                    d, pred[k] = v - pred[k], v
                    n = _nbits(d)
                    toks.append(("s", ("dc", k), n))
                    if n:
                        toks.append(("b", d if d >= 0 else d - 1 + (1 << n), n))
                else:
                    toks.append(("b", (int(blk[0]) >> al) & 1, 1))
                if se == 0:
                    continue
            k0 = max(ss, 1)
            if ah == 0:  # sequential AC or AC first
                r = 0
                for z in range(k0, se + 1):
                    t = int(blk[ZZ[z]])
                    a = abs(t) >> al
                    if a == 0:
                        r += 1
                        continue
                    if ss > 0:
                        emit_eobrun(k)
                    while r > 15:
                        toks.append(("s", ("ac", k), 0xF0))
                        r -= 16
                    n = a.bit_length()
                    toks.append(("s", ("ac", k), (r << 4) | n))
                    toks.append(("b", a if t > 0 else (~a) & ((1 << n) - 1), n))
                    r = 0
                if r:
                    if ss == 0:
                        toks.append(("s", ("ac", k), 0x00))
                    else:
                        eob[0] += 1
                        if eob[0] == 0x7FFF:
                            emit_eobrun(k)
                continue
            # AC refinement
            absv = [abs(int(blk[ZZ[z]])) >> al for z in range(ss, se + 1)]
            last = max([i for i, a in enumerate(absv) if a == 1], default=-1)
            r, br = 0, []
            for i, a in enumerate(absv):
                if a == 0:
                    r += 1
                    continue
                while r > 15 and i <= last:
                    emit_eobrun(k)
                    toks.append(("s", ("ac", k), 0xF0))
                    r -= 16
                    toks.extend(("b", b, 1) for b in br)
                    br = []
                if a > 1:
                    br.append(a & 1)
                    continue
                emit_eobrun(k)
                toks.append(("s", ("ac", k), (r << 4) | 1))
                toks.append(("b", 1 if blk[ZZ[ss + i]] > 0 else 0, 1))
                toks.extend(("b", b, 1) for b in br)
                br, r = [], 0
            if r or br:
                eob[0] += 1
                eob[1] += br
                if eob[0] == 0x7FFF or len(eob[1]) > 1000 - 64 + 1:
                    emit_eobrun(k)
    emit_eobrun(0)
    return toks


def transcode(data, script, progressive=True, dri=0):
    """-> a JPEG file with the coefficients of `data` (a baseline file) coded by `script`."""
    from oracle import jpeg_numpy as J

    d = bytes(data)
    hd = J.parse(d)
    coef = J.entropy_decode(d, hd)
    out = bytearray(b"\xff\xd8")
    p = 2
    while True:  # keep APPn / COM / DQT, rewrite SOF, drop DHT / DRI
        m, L = d[p + 1], (d[p + 2] << 8) | d[p + 3]
        seg = d[p:p + 2 + L]
        p += 2 + L
        if m == 0xDA:
            break
        if m in (0xC0, 0xC1):
            out += bytes([0xFF, 0xC2 if progressive else 0xC0]) + seg[2:]
            if dri:
                out += b"\xff\xdd\x00\x04" + dri.to_bytes(2, "big")
        elif m not in (0xC4, 0xDD):
            out += seg
    for comps, ss, se, ah, al in script:
        toks = _scan_tokens(coef, hd, comps, ss, se, ah, al, dri)
        keys = sorted({t[1] for t in toks if t[0] == "s"})
        tables, ids, dht = {}, {}, bytearray()
        for key in keys:
            freq = [0] * 256
            for t in toks:
                if t[0] == "s" and t[1] == key:
                    freq[t[2]] += 1
            counts, syms = _optimal_table(freq)
            tid = comps.index(comps[key[1]]) if len(comps) > 1 else 0
            ids[key] = tid
            tables[key] = _codes(counts, syms)
            dht += bytes([(0 if key[0] == "dc" else 0x10) | tid]) + bytes(counts) + bytes(syms)
        if dht:
            out += b"\xff\xc4" + (len(dht) + 2).to_bytes(2, "big") + dht
        sos = bytes([len(comps)])
        for k, c in enumerate(comps):
            td, ta = (ids.get(("dc", k), 0), ids.get(("ac", k), 0))
            sos += bytes([hd["comps"][c][0], (td << 4) | ta])
        sos += bytes([ss, se, (ah << 4) | al])
        out += b"\xff\xda" + (len(sos) + 2).to_bytes(2, "big") + sos
        w, rst = _Writer(), 0
        for t in toks:
            if t[0] == "s":
                code, n = tables[t[1]][t[2]]
                w.bits(code, n)
            elif t[0] == "b":
                w.bits(t[1], t[2])
            else:
                w.flush()
                w.out += bytes([0xFF, 0xD0 + rst % 8])
                rst += 1
        w.flush()
        out += w.out
    return bytes(out + b"\xff\xd9")


def transcoded(seed=21):
    """-> list of (name, bytes): every script on noise in the four samplings and in grayscale, with and without restart
    intervals (counted in the scan's MCUs: single blocks when it is not interleaved)."""
    rng = np.random.default_rng(seed)
    out = []
    for samp in list(SAMPLINGS) + ["gray"]:
        img = content("noise", 37, 61, rng)
        b = cv2_jpeg(img[:, :, 0].copy(), 90) if samp == "gray" else cv2_jpeg(img, 90, samp)
        for name, script in SCRIPTS.items():
            for dri in (0, 3):
                out.append(("tc_%s_%s_rst%d" % (name, samp, dri),
                            transcode(b, for_components(script, 1 if samp == "gray" else 3), name not in SEQUENTIAL, dri)))
    return out


def eob_32767():
    """A flat 1456x1456 grayscale frame (33124 blocks without AC) in a DC + AC 1..63 script: an EOB run of 32767 blocks,
    then one of 357."""
    b = cv2_jpeg(np.full((1456, 1456), 77, np.uint8), 90)
    t = transcode(b, [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 0)])
    return t


def scan_cap(n):
    """A grayscale file with n = 64 or 65 scans: DC (at Al = 1 plus its refinement when n = 65), then one scan per AC
    coefficient."""
    b = cv2_jpeg(content("noise", 16, 24, np.random.default_rng(8))[:, :, 0].copy(), 90)
    dc = [((0,), 0, 0, 0, 1), ((0,), 0, 0, 1, 0)] if n == 65 else [((0,), 0, 0, 0, 0)]
    return transcode(b, dc + [((0,), k, k, 0, 0) for k in range(1, 64)])


def eob_flood(symbols=70000):
    """A 16x16 grayscale progressive file whose AC scan is `symbols` EOB14 runs of 32767 blocks, 15 bits each: libjpeg
    stops after the first (the scan holds 4 blocks) and ignores the rest, while summing the runs passes 2^31 blocks."""
    b = transcode(cv2_jpeg(np.full((16, 16), 90, np.uint8), 90), [((0,), 0, 0, 0, 0)])[:-2]
    dht = b"\xff\xc4\x00\x14\x10" + bytes([1] + [0] * 15) + b"\xe0"  # one code, "0", for EOB14
    sos = b"\xff\xda\x00\x08\x01" + bytes([b[b.find(b"\xff\xc2") + 10], 0x00]) + bytes([1, 63, 0])
    w = _Writer()
    for _ in range(symbols):
        w.bits(0x3FFF, 15)  # "0" + 14 one bits
    w.flush()
    return b + dht + sos + bytes(w.out) + b"\xff\xd9"
