"""Pure-Python inflate that reports the block structure of a zlib stream, and the block finder's rule of png.cu restated.

blocks(z) -> (data, [Block]) walks a whole zlib stream (header, blocks, Adler-32 not checked) and raises ValueError where
zlib refuses the stream or a distance reaches past the window its header declares.  finder_accepts(z, bit) is
find_kernel's test of whether a dynamic block header could start at bit `bit` of the stream, candidates(z) every bit where
it holds, and predicted_stats(z) the inflate counters (smapb_png_inflate_stats) a decode of the stream alone reports."""
from collections import namedtuple

import numpy as np

# syms: the literal and length symbols of a fixed or dynamic block, its end-of-block code excluded (0 for stored blocks)
Block = namedtuple("Block", "type start end out_len final syms")
COUNT_MAX_SYMBOLS = 1 << 16  # png.cu: count_kernel leaves a longer block to the serial walk

CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]


class Bits:
    """LSB-first bit reader over bytes; reading past the end raises ValueError."""

    def __init__(self, data):
        self.d = bytes(data) + bytes(4)
        self.n = 8 * len(data)
        self.p = 0

    def peek(self, k):  # k <= 25; zeros past the end
        i = self.p >> 3
        return (int.from_bytes(self.d[i:i + 4], "little") >> (self.p & 7)) & ((1 << k) - 1)

    def get(self, k):
        if self.p + k > self.n:
            raise ValueError("stream ends early")
        r = self.peek(k)
        self.p += k
        return r


def code(lens):
    """Canonical code as (count per length, symbols in code order); ValueError where zlib's inflate_table fails."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    left, maxl = 1, max(lens) if lens else 0
    for l in range(1, 16):
        left = (left << 1) - count[l]
        if left < 0:
            raise ValueError("over-subscribed code")
    if left > 0 and maxl > 1:
        raise ValueError("incomplete code")
    return count, [s for l in range(1, 16) for s, sl in enumerate(lens) if sl == l]


def decode_sym(b, tab):
    count, syms = tab
    v = b.peek(15)
    c = first = index = 0
    for l in range(1, 16):
        c |= (v >> (l - 1)) & 1
        if c - count[l] < first:
            b.get(l)
            return syms[index + c - first]
        index += count[l]
        first = (first + count[l]) << 1
        c <<= 1
    raise ValueError("invalid code")


def dyn_lengths(b, strict=False):
    """Reads HLIT, HDIST, HCLEN and the code lengths (the 3 header bits already read) -> (lit lengths, dist lengths)."""
    hlit, hdist, hclen = b.get(5), b.get(5), b.get(4) + 4
    if hlit > 29 or hdist > 29:
        raise ValueError("too many length or distance symbols")
    cl = [0] * 19
    for i in range(hclen):
        cl[CLORDER[i]] = b.get(3)
    if sum(1 << (7 - l) for l in cl if l) != 128:
        raise ValueError("invalid code lengths set")  # zlib needs a complete code-length code
    ct = code(cl)
    nl, total, lens = hlit + 257, hlit + 257 + hdist + 1, []
    while len(lens) < total:
        s = decode_sym(b, ct)
        if s < 16:
            lens.append(s)
            continue
        if s == 16:
            if not lens:
                raise ValueError("invalid bit length repeat")
            rep, val = 3 + b.get(2), lens[-1]
        elif s == 17:
            rep, val = 3 + b.get(3), 0
        else:
            rep, val = 11 + b.get(7), 0
        if len(lens) + rep > total:
            raise ValueError("invalid bit length repeat")
        lens += [val] * rep
    if lens[256] == 0:
        raise ValueError("missing end-of-block")
    if strict and sum(1 << (15 - l) for l in lens[:nl] if l) != 1 << 15:
        raise ValueError("incomplete literal/length code")
    return lens[:nl], lens[nl:]


def blocks(z):
    """-> (inflated bytes, [Block]) with bit positions relative to the stream's first byte."""
    b = Bits(z)
    b.get(16)
    wsize = 1 << ((z[0] >> 4) + 8)
    out, res = bytearray(), []
    while True:
        start = b.p
        final, t = b.get(1), b.get(2)
        n0, syms = len(out), 0
        if t == 0:
            b.p = (b.p + 7) & ~7
            ln, nln = b.get(16), b.get(16)
            if ln != (~nln & 0xffff):
                raise ValueError("invalid stored block lengths")
            b.get(8 * ln)  # bounds check only
            out += z[b.p // 8 - ln:b.p // 8]
        elif t == 3:
            raise ValueError("invalid block type")
        else:
            if t == 1:
                ll, dl = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, [5] * 32  # 30 and 31 complete the code, decoding them fails
            else:
                ll, dl = dyn_lengths(b)
            lt, dt = code(ll), code(dl)
            while True:
                s = decode_sym(b, lt)
                syms += s != 256
                if s < 256:
                    out.append(s)
                    continue
                if s == 256:
                    break
                s -= 257
                if s >= 29:
                    raise ValueError("invalid literal/length code")
                ln = LBASE[s] + b.get(LEXT[s])
                d = decode_sym(b, dt)
                if d >= 30:
                    raise ValueError("invalid distance code")
                dist = DBASE[d] + b.get(DEXT[d])
                if dist > wsize or dist > len(out):
                    raise ValueError("invalid distance too far back")
                for _ in range(ln):
                    out.append(out[-dist])
        res.append(Block(t, start, b.p, len(out) - n0, final, syms))
        if final:
            return bytes(out), res


def finder_accepts(z, bit):
    """find_kernel's rule at bit `bit`: BTYPE 2, HLIT and HDIST <= 29, a complete code-length code, code lengths that decode
    inside the stream, a complete literal/length code with symbol 256."""
    b = Bits(z)
    b.p = bit
    try:
        b.get(1)
        if b.get(2) != 2:
            return False
        dyn_lengths(b, strict=True)
        return True
    except ValueError:
        return False


def candidates(z):
    """Every bit offset (from 16 on) where finder_accepts(z, bit) holds, ascending.  numpy tests the first 17 header bits and
    the code-length code's Kraft sum at every offset; the few survivors are decoded on one shared Bits."""
    n = 8 * len(z)
    if n < 33:
        return []
    bits = np.unpackbits(np.frombuffer(bytes(z) + bytes(16), np.uint8), bitorder="little").astype(np.int64)

    def field(pos, k):
        v = np.zeros(len(pos), np.int64)
        for i in range(k):
            v |= bits[pos + i] << i
        return v

    pos = np.arange(16, n - 16, dtype=np.int64)  # bit + 17 <= n
    v = field(pos, 17)
    pos = pos[(((v >> 1) & 3) == 2) & (((v >> 3) & 31) <= 29) & (((v >> 8) & 31) <= 29)]
    hclen = field(pos + 13, 4) + 4
    kr = np.zeros(len(pos), np.int64)
    for i in range(19):
        l = field(pos + 17 + 3 * i, 3)
        kr += np.where((i < hclen) & (l > 0), 1 << (7 - l), 0)
    pos = pos[(kr == 128) & (pos + 17 + 3 * hclen <= n)]
    b = Bits(z)
    out = []
    for p in pos.tolist():
        b.p = p + 3
        try:
            dyn_lengths(b, strict=True)
            out.append(p)
        except ValueError:
            pass
    return out


def predicted_stats(z, max_blocks=None):
    """The counters of a decode of stream z alone when the candidates fit their slots: candidates = candidates(z);
    confirmed = chained dynamic blocks among them with at most COUNT_MAX_SYMBOLS symbols; serial = the other chained
    blocks; false positives = candidates that are not chained blocks.  max_blocks: the chain stops after that many."""
    cand = candidates(z)
    chained = blocks(z)[1][:max_blocks]
    cs = set(cand)
    hit = [k for k in chained if k.type == 2 and k.start in cs]
    confirmed = sum(k.syms <= COUNT_MAX_SYMBOLS for k in hit)
    return dict(candidates=len(cand), false_positives=len(cand) - len(hit), confirmed=confirmed,
                serial=len(chained) - confirmed)
