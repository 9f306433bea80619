"""CPU restatement of the GPU JPEG encoder (smap_b200/csrc/jpeg_enc.cu), pinned byte for byte against
cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, q]) (opencv-python's bundled libjpeg-turbo) by tests/test_jpeg_encode_cpu.py.

The stream is cv2's default one: baseline Huffman (SOF0), 3 components with 4:2:0 sampling (luma 2x2, chroma 1x1), the
standard tables of ITU-T T.81 Annex K scaled by the IJG quality rule with baseline clamping, no restart interval, and the
markers SOI, APP0 (JFIF 1.01, density 1:1), DQT x2, SOF0, DHT x4 (DC0, AC0, DC1, AC1), SOS, entropy data, EOI.

    ycc = colour_planes(bgr)          # fixed-point RGB -> YCbCr, h2v2 downsampling, edge replication to the MCU grid
    coef = forward_blocks(ycc, q)     # level shift, accurate-integer FDCT, quantisation -> int [blocks, 64] (zigzag)
    data = entropy_code(coef)         # DC prediction, run/size tokens, MSB-first packing, 1-bit padding, 0xFF stuffing
    encode(bgr, q) does all three and adds the headers.

The arithmetic is the published one: the JFIF YCbCr equations with 16-bit fixed-point constants (Cb/Cr rounded with
1/2 - epsilon), the 2x2 box downsampler whose rounding bias alternates 1, 2 along each row, and the Loeffler-Ligtenberg-
Moschytz 8-point DCT in 13-bit fixed point with 2 extra pass-1 bits (the IJG "islow" method).  Quantisation divides by
8 * Q (the FDCT's output scale) rounding half away from zero: tests/test_jpeg_encode_cpu.py checks at every quality
1..100 that libjpeg-turbo's reciprocal multiplication gives the same integers.
"""
import numpy as np

# ITU-T T.81 Annex K.1 quantisation tables, zigzag order (as DQT stores them)
BASE_Q = np.array([
    [16, 11, 12, 14, 12, 10, 16, 14, 13, 14, 18, 17, 16, 19, 24, 40, 26, 24, 22, 22, 24, 49, 35, 37, 29, 40, 58, 51, 61, 60,
     57, 51, 56, 55, 64, 72, 92, 78, 64, 68, 87, 69, 55, 56, 80, 109, 81, 87, 95, 98, 103, 104, 103, 62, 77, 113, 121, 112,
     100, 120, 92, 101, 103, 99],
    [17, 18, 18, 24, 21, 24, 47, 26, 26, 47, 99, 66, 56, 66, 99] + [99] * 49], np.int64)

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63])

# ITU-T T.81 Annex K.3 Huffman tables: (code-length counts 1..16, symbols)
DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
DC_VALS = (list(range(12)), list(range(12)))
AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77])
AC_VALS = (
    list(bytes.fromhex("01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a"
                       "3435363738393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a929394"
                       "95969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8"
                       "e9eaf1f2f3f4f5f6f7f8f9fa")),
    list(bytes.fromhex("000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728"
                       "292a35363738393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92"
                       "939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7"
                       "e8e9eaf2f3f4f5f6f7f8f9fa")))
assert len(AC_VALS[0]) == 162 and len(AC_VALS[1]) == 162

# worst-case entropy-coded bits of one block under these tables: the longest DC token (category 11 with its code) and
# 63 tokens of run 0 / size 10 (a run token, ZRL or EOB never costs more per coefficient it covers)
BLOCK_BITS_MAX = 22 + 63 * 26


def quant_tables(q):
    """jpeg_set_quality(q, force_baseline=TRUE) -> int [2, 64] (luma, chroma), zigzag order."""
    if not 1 <= q <= 100:
        raise ValueError("quality must be in 1..100")
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((BASE_Q * scale + 50) // 100, 1, 255)


def huff_codes(bits, vals):
    """Canonical Huffman codes -> (code[256], length[256]) indexed by symbol."""
    code, length = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            code[vals[k]], length[vals[k]] = c, n
            c += 1
            k += 1
        c <<= 1
    return code, length


def header(q, h, w):
    """SOI .. SOS of the stream for a w x h frame at quality q."""
    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body

    qt = quant_tables(q)
    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(2):
        out += seg(0xDB, bytes([t]) + bytes(qt[t].astype(np.uint8)))
    out += seg(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for t in range(2):
        out += seg(0xC4, bytes([t]) + bytes(DC_BITS[t]) + bytes(DC_VALS[t]))
        out += seg(0xC4, bytes([0x10 | t]) + bytes(AC_BITS[t]) + bytes(AC_VALS[t]))
    return out + seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


# ---- colour ------------------------------------------------------------------------------------------------------------
def _fix(x):
    return int(x * 65536 + 0.5)


def rgb_to_ycc(bgr):
    """uint8 BGR [..., 3] -> int Y, Cb, Cr (16-bit fixed point, Cb/Cr rounded with 1/2 - epsilon)."""
    b, g, r = (bgr[..., c].astype(np.int64) for c in range(3))
    half = 1 << 15
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + (128 << 16) + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + (128 << 16) + half - 1) >> 16
    return y, cb, cr


def mcu_grid(h, w):
    """-> (MCU columns, MCU rows, luma block columns, luma block rows) of a w x h frame."""
    return (w + 15) // 16, (h + 15) // 16, (w + 7) // 8, (h + 7) // 8


def colour_planes(bgr):
    """uint8 BGR [H,W,3] -> (Y [16*my, 16*mx], Cb, Cr [8*my, 8*mx]) as the encoder's blocks read them.  Luma: the frame with
    its last column and row replicated.  Chroma: the frame replicated to the MCU width and to an even height, 2x2 means
    with the alternating bias, then its last chroma row replicated down to the MCU height."""
    H, W = bgr.shape[:2]
    mx, my, _, _ = mcu_grid(H, W)
    y, cb, cr = rgb_to_ycc(np.pad(bgr, ((0, 16 * my - H), (0, 16 * mx - W), (0, 0)), mode="edge"))
    ch = (H + 1) // 2
    bias = np.tile([1, 2], 4 * mx)[None, :]
    out = [y]
    for c in (cb, cr):
        c = c[:2 * ch]
        d = (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + bias) >> 2
        out.append(np.pad(d, ((0, 8 * my - ch), (0, 0)), mode="edge"))
    return tuple(out)


# ---- forward DCT and quantisation -----------------------------------------------------------------------------------
_C = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
          c2053=16819, c2562=20995, c3072=25172)


def _fdct_1d(d, shift_odd, first):
    """One pass of the islow FDCT along the last axis of d (int64 [..., 8])."""
    c = _C
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2

    def ds(x, n):
        return (x + (1 << (n - 1))) >> n

    o = np.empty_like(d)
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        o[..., 0], o[..., 4] = ds(t10 + t11, 2), ds(t10 - t11, 2)
    z1 = (t12 + t13) * c["c0541"]
    o[..., 2] = ds(z1 + t13 * c["c0765"], shift_odd)
    o[..., 6] = ds(z1 - t12 * c["c1847"], shift_odd)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * c["c1175"]
    t4, t5, t6, t7 = t4 * c["c0298"], t5 * c["c2053"], t6 * c["c3072"], t7 * c["c1501"]
    z1, z2 = z1 * -c["c0899"], z2 * -c["c2562"]
    z3, z4 = z3 * -c["c1961"] + z5, z4 * -c["c0390"] + z5
    o[..., 7] = ds(t4 + z1 + z3, shift_odd)
    o[..., 5] = ds(t5 + z2 + z4, shift_odd)
    o[..., 3] = ds(t6 + z2 + z3, shift_odd)
    o[..., 1] = ds(t7 + z1 + z4, shift_odd)
    return o


def fdct(blocks):
    """int [n, 8, 8] level-shifted samples -> int64 [n, 8, 8] FDCT output (8x the orthonormal DCT)."""
    d = _fdct_1d(blocks.astype(np.int64), 13 - 2, True)
    d = _fdct_1d(d.transpose(0, 2, 1), 13 + 2, False)
    return d.transpose(0, 2, 1)


def quantise(coef, qt):
    """FDCT output (natural order) / (8 * qt) rounded half away from zero -> zigzag order."""
    z = coef.reshape(coef.shape[0], 64)[:, ZIGZAG]
    div = 8 * qt[None, :]
    a = (np.abs(z) + div // 2) // div
    return np.where(z < 0, -a, a)


def _blocks(plane):
    r, c = plane.shape
    return plane.reshape(r // 8, 8, c // 8, 8).transpose(0, 2, 1, 3)  # [block row, block col, 8, 8]


def forward_blocks(planes, q, h, w):
    """Colour planes -> int64 [my * mx * 6, 64] quantised coefficients in scan order (per MCU: Y00 Y01 Y10 Y11 Cb Cr),
    zigzag order.  Luma blocks past the frame's own block grid are libjpeg's dummy blocks: zero AC and the DC of the
    block before them in the MCU."""
    qt = quant_tables(q)
    mx, my, bw, bh = mcu_grid(h, w)
    Y, Cb, Cr = planes
    yq = quantise(fdct(_blocks(Y).reshape(-1, 8, 8) - 128), qt[0]).reshape(2 * my, 2 * mx, 64)
    cq = [quantise(fdct(_blocks(c).reshape(-1, 8, 8) - 128), qt[1]).reshape(my, mx, 64) for c in (Cb, Cr)]
    mcu = yq.reshape(my, 2, mx, 2, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, 4, 64).copy()
    by, bx = np.arange(my)[:, None, None] * 2 + np.array([0, 0, 1, 1]), np.arange(mx)[None, :, None] * 2 + np.array([0, 1, 0, 1])
    real = (by < bh) & (bx < bw)
    for k in range(1, 4):  # block 0 of an MCU is always inside the frame
        d = ~real[..., k]
        mcu[d, k, :] = 0
        mcu[d, k, 0] = mcu[d, k - 1, 0]
    out = np.concatenate([mcu, cq[0][:, :, None], cq[1][:, :, None]], axis=2)
    return out.reshape(-1, 64)


# ---- entropy coding ---------------------------------------------------------------------------------------------------
def _category(v):
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while True:
        m = a >> n > 0
        if not m.any():
            return n
        n += m


def _extra(v, s):
    return np.where(v < 0, v + (1 << s) - 1, v) & ((1 << s) - 1)


def tokens(coef):
    """Scan-order coefficients -> (value, length) of every token in stream order: per block its DC difference, then
    (ZRL*, run/size) per nonzero AC coefficient and an EOB when the block ends in zeros, codes and extra bits merged."""
    n = coef.shape[0]
    comp = np.tile([0, 0, 0, 0, 1, 2], n // 6)
    tab = np.where(comp == 0, 0, 1)
    dc = coef[:, 0]
    pred = np.zeros(n, np.int64)
    for c in range(3):
        i = np.flatnonzero(comp == c)
        pred[i[1:]] = dc[i[:-1]]
    diff = dc - pred
    dcode = [huff_codes(DC_BITS[t], DC_VALS[t]) for t in range(2)]
    acode = [huff_codes(AC_BITS[t], AC_VALS[t]) for t in range(2)]
    s = _category(diff)
    dcc = np.where(tab == 0, dcode[0][0][s], dcode[1][0][s])
    dcl = np.where(tab == 0, dcode[0][1][s], dcode[1][1][s])
    keys, vals, lens = [np.arange(n) * 256], [(dcc << s) | _extra(diff, s)], [dcl + s]
    b, k = np.nonzero(coef[:, 1:])
    k = k + 1
    first = np.r_[True, b[1:] != b[:-1]] if len(b) else np.zeros(0, bool)
    prev = np.where(first, 0, np.r_[0, k[:-1]])
    run = k - prev - 1
    v = coef[b, k]
    sz = _category(v)
    sym = ((run & 15) << 4) | sz
    t = tab[b]
    ac_c = np.where(t == 0, acode[0][0][sym], acode[1][0][sym])
    ac_l = np.where(t == 0, acode[0][1][sym], acode[1][1][sym])
    keys.append(b * 256 + 2 * k)
    vals.append((ac_c << sz) | _extra(v, sz))
    lens.append(ac_l + sz)
    nz = run >> 4
    zi = np.repeat(np.arange(len(b)), nz)
    keys.append(b[zi] * 256 + 2 * k[zi] - 1)
    vals.append(np.where(t[zi] == 0, acode[0][0][0xF0], acode[1][0][0xF0]))
    lens.append(np.where(t[zi] == 0, acode[0][1][0xF0], acode[1][1][0xF0]))
    last = np.full(n, 0, np.int64)
    if len(b):
        last[b] = k  # k ascends within a block, so the last write is the block's last nonzero
    e = np.flatnonzero(last < 63)
    keys.append(e * 256 + 255)
    vals.append(np.where(tab[e] == 0, acode[0][0][0], acode[1][0][0]))
    lens.append(np.where(tab[e] == 0, acode[0][1][0], acode[1][1][0]))
    order = np.argsort(np.concatenate(keys), kind="stable")
    return np.concatenate(vals)[order], np.concatenate(lens)[order]


def pack(vals, lens):
    """MSB-first packing of the tokens, the last byte padded with 1-bits -> (bytes, number of bits before padding)."""
    off = np.cumsum(lens) - lens
    total = int(off[-1] + lens[-1]) if len(lens) else 0
    words = np.zeros(total // 64 + 2, np.uint64)
    w, r = off // 64, off % 64
    shift = 64 - r - lens  # < 0 when the token spills into the next word
    u = vals.astype(np.uint64)
    hi = np.where(shift >= 0, u << np.maximum(shift, 0).astype(np.uint64), u >> np.maximum(-shift, 0).astype(np.uint64))
    np.add.at(words, w, hi)  # the tokens of a word occupy disjoint bits, so the sum is their OR
    sp = np.flatnonzero(shift < 0)
    lo = (u[sp] & ((np.uint64(1) << (-shift[sp]).astype(np.uint64)) - np.uint64(1))) << (64 + shift[sp]).astype(np.uint64)
    np.add.at(words, w[sp] + 1, lo)
    data = bytearray(words.astype(">u8").tobytes()[:(total + 7) // 8])
    if total % 8:
        data[-1] |= (1 << (8 - total % 8)) - 1
    return bytes(data), total


def stuff(data):
    """0x00 after every 0xFF byte."""
    a = np.frombuffer(data, np.uint8)
    return np.insert(a, np.flatnonzero(a == 0xFF) + 1, 0).tobytes()


def entropy_code(coef):
    return stuff(pack(*tokens(coef))[0])


def encode(bgr, q=95):
    """uint8 BGR [H,W,3] -> the bytes cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, q]) writes."""
    bgr = np.ascontiguousarray(bgr)
    H, W = bgr.shape[:2]
    if not (1 <= H <= 65535 and 1 <= W <= 65535) or bgr.ndim != 3 or bgr.shape[2] != 3 or bgr.dtype != np.uint8:
        raise ValueError("uint8 [H,W,3] expected")
    return header(q, H, W) + entropy_code(forward_blocks(colour_planes(bgr), q, H, W)) + b"\xff\xd9"
