"""Seeded DEFLATE / zlib writer for the PNG decoder's inflate tests (tests/test_png_deflate_cpu.py, test_png_deflate_gpu.py).

zlib's deflate writes a narrow subset of what its inflate accepts; other PNG writers (libdeflate, zopfli, fpnge, fdeflate,
Go's image/png) write the rest.  This writer emits stored, fixed and dynamic blocks over a token list (literals and
length / distance pairs) with the block shapes zlib never writes: dynamic headers from caller-given code lengths with a
chosen HCLEN, with or without repeat codes 16, 17 and 18, and runs that cross from the literal into the distance lengths;
15-bit codes; length 258 as code 284 plus 31 extra bits; matches exactly 32 768 back or back to the first byte; blocks of
more than 65 536 symbols; more blocks than bytes / 8; a chosen zlib window (CINFO); zero-length IDATs.

adversarial() -> [(name, png bytes, expect)], expect one of
  "decode"          the GPU decoder must decode it (to cv2's bytes),
  "device_refuses"  cv2 reads it, but it is past one of the GPU decoder's two documented limits: more blocks than
                    zlen / 8 + 64, or a match reaching past the window the zlib header declares,
  "both_refuse"     cv2 refuses it too.
cases() returns the same files as Case records with the stream, the scanline bytes and the intended block structure."""
import heapq
import zlib
from collections import namedtuple

import numpy as np

from png_corpus import samples, scanlines, write_png

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32

COUNT_MAX_SYMBOLS = 1 << 16  # png.cu: a candidate block with more symbols is left to the serial walk

Rec = namedtuple("Rec", "type start syms final")  # the intended block structure: start bit within the zlib stream
Case = namedtuple("Case", "name png expect z raw blocks ref_png")


def blk_cap(zlen):
    """Block records png.cu reserves per image: more blocks than this leave the file to cv2."""
    return zlen // 8 + 64


def cand_cap(zlens):
    """Candidate slots png.cu allots a batch whose zlib streams have these lengths."""
    return sum((n + 16 + 15) // 16 * 16 for n in zlens) // 64 + 4096


class BitWriter:
    """LSB-first bit writer: a bytearray and a bit buffer of fewer than 8 pending bits."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    @property
    def pos(self):
        return 8 * len(self.out) + self.n

    def put(self, v, k):
        self.acc |= (v & ((1 << k) - 1)) << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def put_code(self, code, length):  # Huffman codes go most significant bit first
        self.put(int(format(code, "0%db" % length)[::-1], 2), length)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def getvalue(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lens):
    """Canonical codes of the lengths (0 = unused)."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    nxt, c = [0] * 16, 0
    for l in range(1, 16):
        c = (c + count[l - 1]) << 1
        nxt[l] = c
    codes = [0] * len(lens)
    for s, l in enumerate(lens):
        if l:
            codes[s] = nxt[l]
            nxt[l] += 1
    return codes


def kraft(lens, limit=15):
    return sum(1 << (limit - l) for l in lens if l)


def huffman_lengths(freq, limit):
    """Huffman code lengths of the symbols with freq > 0, capped at `limit` and kept complete (two symbols at least)."""
    lens = [0] * len(freq)
    used = [s for s, f in enumerate(freq) if f > 0]
    if len(used) < 2:
        for s in (used + [s for s in range(len(freq)) if s not in used])[:2]:
            lens[s] = 1
        return lens
    heap = [(freq[s], s, [s]) for s in used]
    heapq.heapify(heap)
    k = len(freq)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            lens[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    if max(lens) > limit:
        lens = [min(l, limit) for l in lens]
        full = 1 << limit
        by_freq = sorted(used, key=lambda s: (freq[s], -s))
        while kraft(lens, limit) > full:  # lengthen the rarest symbol that can still grow
            s = next(s for s in by_freq if lens[s] < limit)
            lens[s] += 1
        for s in reversed(by_freq):  # then shorten the most frequent ones while the code stays a prefix code
            while lens[s] > 1 and kraft(lens, limit) + (1 << (limit - lens[s])) <= full:
                lens[s] -= 1
    assert kraft(lens, limit) == 1 << limit
    return lens


def fib_freq(symbols, n):
    """Fibonacci-like frequencies over the given symbols: codes as long as the length limit allows."""
    f = [0] * n
    a, b = 1, 1
    for s in symbols:
        f[s] = a
        a, b = b, a + b
    return f


# ---- tokens --------------------------------------------------------------------------------------------------------------
# A token is a literal byte (int) or a match (lsym, lextra, dsym, dextra, length, dist).
def len_sym(n, use284=False):
    if n == 258 and use284:
        return 284, 31
    for i in range(28, -1, -1):
        if LBASE[i] <= n and n - LBASE[i] < (1 << LEXT[i]) and (i < 28 or n == 258):
            return 257 + i, n - LBASE[i]
    raise ValueError(n)


def dist_sym(d):
    for i in range(29, -1, -1):
        if DBASE[i] <= d:
            assert d - DBASE[i] < 1 << DEXT[i]
            return i, d - DBASE[i]
    raise ValueError(d)


def match(n, d, use284=False):
    ls, le = len_sym(n, use284)
    ds, de = dist_sym(d)
    return (ls, le, ds, de, n, d)


def lz77(raw, lo, hi, maxdist=32768, maxlen=258, mindist=1, only_dist=None, forced=None, greedy=True, use284=False):
    """Tokens for raw[lo:hi]: greedy matches over the 8 latest positions with the same 3 bytes (none if not greedy), within
    maxdist back from any earlier byte of raw (before lo too) and inside [lo, hi); forced = {pos: (length, dist)}."""
    forced = forced or {}
    raw = bytes(raw)
    table = {}
    toks = []
    if greedy:
        for p in range(max(0, lo - maxdist), lo):
            table.setdefault(raw[p:p + 3], []).append(p)
    p = lo
    while p < hi:
        best, bd = 0, 0
        if p in forced:
            best, bd = forced[p]
            assert p + best <= hi and all(raw[p + k] == raw[p + k - bd] for k in range(best)), (p, best, bd)
        elif greedy and p + 3 <= hi:
            cands = [only_dist] if only_dist else reversed(table.get(raw[p:p + 3], [])[-8:])
            for c in cands:
                d = p - c if not only_dist else c
                if not (mindist <= d <= min(maxdist, p)):
                    continue
                n, top = 0, min(maxlen, hi - p)
                while n < top and raw[p + n] == raw[p + n - d]:
                    n += 1
                if n > best:
                    best, bd = n, d
        if best >= 3:
            toks.append(match(best, bd, use284))
            step = best
        else:
            toks.append(raw[p])
            step = 1
        if greedy:
            for q in range(p, p + step):
                table.setdefault(raw[q:q + 3], []).append(q)
        p += step
    return toks


def rle(lens, use16=True, use17=True, use18=True):
    """Code-length symbols (sym, extra bits, extra value, run length) for a list of lengths."""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while use18 and run >= 11:
                k = min(run, 138)
                out.append((18, 7, k - 11, k))
                run -= k
            while use17 and run >= 3:
                k = min(run, 10)
                out.append((17, 3, k - 3, k))
                run -= k
            out += [(0, 0, 0, 1)] * run
        else:
            out.append((v, 0, 0, 1))
            run -= 1
            while use16 and run >= 3:
                k = min(run, 6)
                out.append((16, 2, k - 3, k))
                run -= k
            out += [(v, 0, 0, 1)] * run
    return out


class Deflate:
    """Builds one DEFLATE stream block by block; `out` is what it inflates to, `recs` its block structure."""

    def __init__(self):
        self.w = BitWriter()
        self.out = bytearray()
        self.recs = []
        self.crossing = []  # per dynamic block: True when a repeat code crosses from the literal into the distance lengths

    def _rec(self, t, syms, final):
        self.recs.append(Rec(t, 16 + self.w.pos, syms, final))

    def _expand(self, toks):
        for t in toks:
            if isinstance(t, int):
                self.out.append(t)
            else:
                n, d = t[4], t[5]
                for _ in range(n):
                    self.out.append(self.out[-d] if d <= len(self.out) else 0)

    def stored(self, data, final=False):
        assert len(data) < 65536
        self._rec(0, 0, final)
        self.w.put(final, 1)
        self.w.put(0, 2)
        self.w.align()
        self.w.put(len(data), 16)
        self.w.put(len(data) ^ 0xffff, 16)
        self.w.out += data
        self.out += data

    def _data(self, toks, lens_l, lens_d):
        cl, cd = canonical(lens_l), canonical(lens_d)
        for t in toks:
            if isinstance(t, int):
                assert lens_l[t], t
                self.w.put_code(cl[t], lens_l[t])
            else:
                ls, le, ds, de = t[:4]
                assert lens_l[ls] and lens_d[ds], t
                self.w.put_code(cl[ls], lens_l[ls])
                self.w.put(le, LEXT[ls - 257])
                self.w.put_code(cd[ds], lens_d[ds])
                self.w.put(de, DEXT[ds] if ds < 30 else 13)
        self.w.put_code(cl[256], lens_l[256])
        self._expand(toks)

    def fixed(self, toks, final=False):
        self._rec(1, len(toks), final)
        self.w.put(final, 1)
        self.w.put(1, 2)
        self._data(toks, FIXED_LIT, FIXED_DIST)

    def dynamic(self, toks, final=False, lit=None, dist=None, limit=15, fib=False, nl=None, nd=None, hclen=None,
                use16=True, use17=True, use18=True, joint=False):
        """lit / dist: explicit code lengths (else Huffman lengths of the tokens' frequencies, Fibonacci-like ones with
        fib=True, capped at `limit`; "none" = no distance code, "one" = a single 1-bit distance code).  nl / nd / hclen:
        at least this many lengths.  joint: one run-length sequence over both lists (repeats may cross into the
        distance lengths), else one per list as zlib writes them."""
        fl, fd = [0] * 286, [0] * 30
        for t in toks:
            if isinstance(t, int):
                fl[t] += 1
            else:
                fl[t[0]] += 1
                fd[t[2]] += 1
        fl[256] += 1
        if lit is None:
            used = [s for s in range(286) if fl[s]]
            lit = huffman_lengths(fib_freq(used, 286) if fib else fl, limit)
        if dist is None or dist in ("none", "one"):
            used = [s for s in range(30) if fd[s]]
            if dist == "none":
                assert not used
                dist = [0]
            elif dist == "one":
                assert len(used) <= 1
                dist = [0] * 30
                dist[used[0] if used else 0] = 1
            else:
                dist = huffman_lengths(fib_freq(used, 30) if fib else fd, limit)
        lit, dist = list(lit), list(dist)
        n_l = max(257, nl or 0, max(s for s, l in enumerate(lit) if l) + 1)
        n_d = max(1, nd or 0, max([s for s, l in enumerate(dist) if l], default=0) + 1)
        lit = (lit + [0] * 286)[:n_l]
        dist = (dist + [0] * 30)[:n_d]
        if joint:
            seq = rle(lit + dist, use16, use17, use18)
        else:
            seq = rle(lit, use16, use17, use18) + rle(dist, use16, use17, use18)
        at, cross = 0, False
        for s in seq:
            cross |= at < n_l < at + s[3]
            at += s[3]
        cf = [0] * 19
        for s in seq:
            cf[s[0]] += 1
        cll = huffman_lengths(cf, 7)
        h = max(4, hclen or 0, max(i for i in range(19) if cll[CLORDER[i]]) + 1)
        self._rec(2, len(toks), final)
        self.crossing.append(cross)
        w = self.w
        w.put(final, 1)
        w.put(2, 2)
        w.put(n_l - 257, 5)
        w.put(n_d - 1, 5)
        w.put(h - 4, 4)
        for i in range(h):
            w.put(cll[CLORDER[i]], 3)
        clc = canonical(cll)
        for sym, eb, ev, _ in seq:
            w.put_code(clc[sym], cll[sym])
            w.put(ev, eb)
        self._data(toks, lit + [0] * (288 - n_l), dist + [0] * (32 - n_d))

    def zlib(self, cinfo=7, adler_of=None):
        cmf = cinfo << 4 | 8
        flg = 2 << 6
        flg += (31 - (cmf * 256 + flg) % 31) % 31
        a = zlib.adler32(bytes(self.out if adler_of is None else adler_of))
        return bytes([cmf, flg]) + self.w.getvalue() + a.to_bytes(4, "big")


def one_block_zlib(raw):
    """zlib stream of one final dynamic block of literals only, as fpnge-style writers store a whole frame (numpy bit
    packing: a frame is millions of symbols)."""
    a = np.frombuffer(bytes(raw), np.uint8)
    freq = np.bincount(a, minlength=286).tolist()
    freq[256] = 1
    lit = huffman_lengths(freq, 15)
    d = Deflate()
    d.dynamic([], final=True, lit=lit, dist="none")
    head = np.unpackbits(np.frombuffer(d.w.getvalue(), np.uint8), bitorder="little")[:d.w.pos - lit[256]]
    codes = canonical(lit)
    rev = np.array([int(format(c, "0%db" % l)[::-1], 2) if l else 0 for c, l in zip(codes, lit)], np.int64)
    ln = np.array(lit, np.int64)
    parts = [head]
    for lo in range(0, len(a), 1 << 20):
        sym = np.append(a[lo:lo + (1 << 20)], [256] if lo + (1 << 20) >= len(a) else []).astype(np.int64)
        L = ln[sym]
        start = np.repeat(np.cumsum(L) - L, L)
        j = np.arange(int(L.sum())) - start
        parts.append(((np.repeat(rev[sym], L) >> j) & 1).astype(np.uint8))
    body = np.packbits(np.concatenate(parts), bitorder="little").tobytes()
    return bytes([0x78, 0x9c]) + body + zlib.adler32(bytes(raw)).to_bytes(4, "big")


# ---- scanlines -----------------------------------------------------------------------------------------------------------
def gray_rows(rng, rows, w=255, top=256):
    """Scanlines of an 8-bit grey image, filter type 0 on every row, samples below `top`."""
    a = rng.integers(0, top, (rows, w + 1)).astype(np.uint8)
    a[:, 0] = 0
    return bytearray(a.tobytes())


def gray_png(raw, w, z, **kw):
    h = len(raw) // (w + 1)
    assert h * (w + 1) == len(raw)
    return write_png(np.zeros((h, w, 1), np.uint8), 0, 8, z=z, **kw)


def plant(raw, dst, n, d, rowlen):
    """Copies raw[dst - d:dst - d + n] to dst (overlapping copies repeat, as in LZ77), keeping every filter byte <= 4."""
    for k in range(n):
        raw[dst + k] = raw[dst + k - d]
    assert all(raw[r] <= 4 for r in range(0, len(raw), rowlen))
    return {dst: (n, d)}


def case(name, d, raw, w, expect="decode", cinfo=7, ctype=0, depth=8, shape=None, interlace=0, png_kw=None, z=None):
    assert expect != "decode" or bytes(d.out) == bytes(raw), name
    z = d.zlib(cinfo) if z is None else z
    assert expect == "device_refuses" or len(d.recs) <= blk_cap(len(z)), name
    if shape is None:
        png = gray_png(raw, w, z, **(png_kw or {}))
        ref = gray_png(raw, w, zlib.compress(bytes(raw)))
    else:
        s = np.zeros(shape, np.uint16 if depth == 16 else np.uint8)
        png = write_png(s, ctype, depth, interlace, z=z, **(png_kw or {}))
        ref = write_png(s, ctype, depth, interlace, z=zlib.compress(bytes(raw)))
    return Case(name, png, expect, z, bytes(raw), list(d.recs), ref)


# ---- the files -----------------------------------------------------------------------------------------------------------
def _symbol_cap(rng):
    raw = gray_rows(rng, 513)  # 65 536 + 65 537 + 255 bytes
    d = Deflate()
    d.dynamic(list(raw[:65536]))
    d.dynamic(list(raw[65536:131073]))
    d.fixed(list(raw[131073:]), final=True)
    return case("symbols_65536_then_65537", d, raw, 255)


def _empty_fixed_blocks(nblocks, raw):
    d = Deflate()
    for _ in range(nblocks - 1):
        d.fixed([])
    d.stored(bytes(raw), final=True)
    return d


def _block_cap(rng):
    raw = gray_rows(rng, 4, w=4)
    out = []
    d = _empty_fixed_blocks(201, raw)
    out.append(case("partial_flush_200_empty_blocks", d, raw, 4, "device_refuses"))
    for extra, expect in ((0, "decode"), (1, "device_refuses")):
        n = 1
        while True:
            d = _empty_fixed_blocks(n, raw)
            if n == blk_cap(len(d.zlib())) + extra:
                break
            n += 1
        out.append(case("blocks_eq_blk_cap_plus_%d" % extra, d, raw, 4, expect))
    return out


def flood_header():
    """A dynamic block header the finder accepts (literal code {255, 256}, one 1-bit distance code), padded to bytes."""
    d = Deflate()
    d.dynamic([], lit=[0] * 255 + [1, 1], dist=[1])
    return d.w.getvalue()


def _candidate_flood(rng):
    hdr = flood_header()
    rowlen = 20
    rows = 8000  # 160 000 bytes, one header per row
    a = rng.integers(0, 256, (rows, rowlen)).astype(np.uint8)
    a[:, 0] = 0
    a[:, 1:1 + len(hdr)] = np.frombuffer(hdr, np.uint8)
    tail = samples(0, 8, 1500, rowlen - 1, rng)
    raw = bytearray(a.tobytes()) + bytearray(scanlines(tail, 0, 8, 0, lambda r: r % 5))
    d = Deflate()
    flood = rows * rowlen
    for lo in range(0, flood, 60000):
        d.stored(bytes(raw[lo:min(flood, lo + 60000)]))
    step = (len(raw) - flood) // 4
    for k in range(4):
        lo, hi = flood + k * step, (flood + (k + 1) * step if k < 3 else len(raw))
        d.dynamic(lz77(raw, lo, hi, maxdist=4096), final=k == 3)
    return case("candidate_flood", d, raw, rowlen - 1)


def _cross_boundary(rng):
    """Runs of code lengths that cross from the literal lengths into the distance lengths, with codes 16, 17 and 18."""
    raw = gray_rows(rng, 40, top=30)
    out = []
    lit = [5] * 30 + [0] * 226 + [5, 5]  # 30 literals, EOB and length 3: 32 five-bit codes
    toks16 = lz77(raw, 0, len(raw), maxlen=3)
    toks5 = lz77(raw, 0, len(raw), maxlen=3, mindist=5)
    variants = [
        ("cross_boundary_16", toks16, dict(lit=lit, dist=[5] * 28 + [4, 4])),
        ("cross_boundary_17", toks5, dict(lit=lit, nl=262, dist=[0] * 4 + [4] * 6 + [5] * 20, use18=False)),
        ("cross_boundary_18", toks5, dict(lit=lit, nl=286, dist=[0] * 4 + [4] * 6 + [5] * 20)),
    ]
    for name, toks, kw in variants:
        d = Deflate()
        d.dynamic(toks, final=True, joint=True, **kw)
        assert d.crossing == [True], name
        out.append(case(name, d, raw, 255))
    return out


def _unusual_codes(rng):
    out = []
    raw = gray_rows(rng, 30, top=255)  # no byte 255: the HCLEN blocks give it no code
    d = Deflate()
    per = len(raw) // 16
    for k, h in enumerate(range(5, 20)):  # HCLEN 5..19: all-8 literal codes, trailing code-length lengths 0
        d.dynamic(list(raw[k * per:(k + 1) * per]), lit=[8] * 255 + [0, 8], dist="none", hclen=h)
    d.dynamic([], lit=[0] * 256 + [1], dist="none")  # EOB alone: an incomplete code zlib accepts, the finder skips
    d.dynamic(list(raw[15 * per:]), lit=[8] * 255 + [0, 8], dist=[0] * 29 + [1], final=True)  # unused 1-bit dist code
    out.append(case("hclen_5_to_19_eob_only_literal_only", d, raw, 255))

    raw = bytearray(b"".join(bytes([0]) + bytes([(c // 9 + r // 4 * 3) % 251 for c in range(255)]) for r in range(24)))
    d = Deflate()
    toks = lz77(raw, 0, 3000, only_dist=1)
    d.dynamic(toks, dist="one")  # one 1-bit distance code (distance 1)
    toks = lz77(raw, 3000, len(raw), only_dist=256)
    d.dynamic(toks, dist="one", final=True)  # one 1-bit distance code, symbol 15
    out.append(case("single_one_bit_distance_code", d, raw, 255))

    raw = gray_rows(rng, 300, top=256)
    forced = {}
    for k, dd in enumerate(sorted([DBASE[i] + (1 << DEXT[i]) - 1 for i in range(30)] + DBASE)):  # every distance code
        p = 256 * (3 + 4 * k) + 5 + k  # inside a row, so no filter byte is overwritten
        forced.update(plant(raw, p, 12 + k % 20, dd, 256))
    d = Deflate()
    toks = lz77(raw, 0, len(raw), forced=forced, greedy=False)
    h = len(toks) // 2
    d.dynamic(toks[:h], fib=True)
    d.dynamic(toks[h:], fib=True, final=True, use16=False)
    out.append(case("codes_of_15_bits", d, raw, 255))
    return out


def _len258(rng):
    raw = gray_rows(rng, 8) + bytearray(256 * 24)  # zero rows copy as runs of 258
    d = Deflate()
    d.fixed(lz77(raw, 0, 4000, use284=True))
    d.dynamic(lz77(raw, 4000, len(raw), use284=True), final=True)
    assert sum(1 for t in lz77(raw, 0, len(raw), use284=True) if not isinstance(t, int) and t[0] == 284) > 10
    return case("length_258_as_284_plus_31", d, raw, 255)


def _window(rng):
    out = []
    raw = gray_rows(rng, 140)  # 35 840 bytes
    forced = plant(raw, 32768 + 256 * 2, 258, 32768, 256)  # a whole row and two bytes, 32 768 back
    forced.update(plant(raw, 256 * 127, 256, 256 * 127, 256))  # back to the stream's first byte
    d = Deflate()
    d.stored(bytes(raw[:30000]))
    d.fixed(lz77(raw, 30000, 33000, forced=forced, greedy=False))
    d.dynamic(lz77(raw, 33000, len(raw), forced=forced, greedy=False), final=True)
    out.append(case("distance_32768_and_to_the_first_byte", d, raw, 255))

    # markers of markers: each copy's source is the previous copy, two blocks back (row-aligned distances)
    raw = gray_rows(rng, 100)
    forced = {}
    src = 300
    for dst in (6188, 12076, 19244, 25132):
        forced.update(plant(raw, dst, 200, dst - src, 256))
        src = dst
    # overlapping matches (distance < length) that start a block, their source in the block before
    overlaps = (8 * 256 + 20, 15 * 256 + 9, 22 * 256 + 50)
    for at, dd in zip(overlaps, (3, 1, 7)):
        forced.update(plant(raw, at, 180, dd, 256))
    d = Deflate()
    cuts = sorted([0, 2000, 9000, 15000, 22000, 6188, 12076, 19244, 25132, len(raw)] + list(overlaps))
    for k, (lo, hi) in enumerate(zip(cuts, cuts[1:])):
        toks = lz77(raw, lo, hi, forced=forced, greedy=False)
        (d.fixed if k % 3 == 1 else d.dynamic)(toks, final=hi == len(raw))
    out.append(case("markers_of_markers_and_overlaps_across_blocks", d, raw, 255))

    # the declared window: CINFO 0 (256 bytes)
    raw = gray_rows(rng, 4, w=599)
    forced = plant(raw, 600 + 350, 40, 256, 600)
    d = Deflate()
    d.dynamic(lz77(raw, 0, len(raw), forced=forced, greedy=False), final=True)
    out.append(case("cinfo0_distance_256", d, raw, 599, cinfo=0))
    raw = gray_rows(rng, 4, w=599)
    forced = plant(raw, 600 + 350, 40, 300, 600)
    d = Deflate()
    d.dynamic(lz77(raw, 0, len(raw), forced=forced, greedy=False), final=True)
    out.append(case("cinfo0_distance_300", d, raw, 599, "device_refuses", cinfo=0))
    return out


def _alignment(rng):
    """Block headers at every bit offset mod 32, stored blocks after 0 and 7 padding bits, zero-length IDATs."""
    raw = gray_rows(rng, 40, top=256)
    raw[1::2] = bytes(max(144, b) for b in raw[1::2])
    d = Deflate()
    p = i = 0
    seen = {1: set(), 2: set()}
    want0, want7 = True, True
    while len(seen[1]) < 32 or len(seen[2]) < 32 or want0 or want7:
        pos = 16 + d.w.pos
        if want0 and pos % 8 == 5:
            d.stored(bytes(raw[p:p + 50]))
            p, want0 = p + 50, False
        elif want7 and pos % 8 == 6:
            d.stored(bytes(raw[p:p + 51]))
            p, want7 = p + 51, False
        elif i % 4 == 3:
            seen[2].add(pos % 32)
            d.dynamic(list(raw[p:p + 3]))
            p += 3
        else:
            seen[1].add(pos % 32)
            d.fixed([raw[p]])
            p += 1
        i += 1
    d.dynamic(lz77(raw, p, len(raw)), final=True)
    png_kw = dict(split=lambda k: [0, 0, 7, 0, 1, 0][k] if k < 6 else 0 if k % 5 == 0 else 97, empty_after=2)
    return case("headers_at_every_offset_empty_idats", d, raw, 255, png_kw=png_kw)


def _both_refuse(rng):
    out = []
    raw = gray_rows(rng, 2, w=63)
    d = Deflate()
    d.fixed(list(raw[:100]))
    d.fixed([match(3, 101)] + list(raw[103:]), final=True)  # one byte before the stream's first byte
    out.append(case("distance_past_the_first_byte", d, raw, 63, "both_refuse"))
    for ds in (30, 31):
        d = Deflate()
        d.fixed(list(raw[:100]) + [(257, 0, ds, 0, 3, 1)] + list(raw[103:]), final=True)
        out.append(case("fixed_distance_code_%d" % ds, d, raw, 63, "both_refuse"))
    # HCLEN 4: only 16, 17, 18 and 0 have code-length codes, so no length can be non-zero and EOB has none
    d = Deflate()
    w = d.w
    w.put(1, 1), w.put(2, 2), w.put(0, 5), w.put(0, 5), w.put(0, 4)
    cll = [0] * 19
    for s in CLORDER[:4]:
        cll[s] = 2
        w.put(2, 3)
    clc = canonical(cll)
    w.put_code(clc[18], 2), w.put(127, 7), w.put_code(clc[18], 2), w.put(108, 7)  # 138 + 119 zeros: no EOB length
    w.put_code(clc[0], 2)  # the distance length
    d.out = bytearray(raw)
    out.append(case("hclen_4", d, raw, 63, "both_refuse"))
    return out


def _sweep(rng, n):
    """Random files: random geometry (Adam7 and 16-bit among them), block types and splits, codes and windows."""
    from png_corpus import PAIRS

    out = []
    for i in range(n):
        ctype, depth = PAIRS[rng.integers(len(PAIRS))]
        inter = int(rng.integers(2))
        big = i % 25 == 0
        h, w = (int(rng.integers(60, 90)), int(rng.integers(60, 90))) if big else (int(rng.integers(1, 24)),
                                                                                    int(rng.integers(1, 24)))
        s = samples(ctype, depth, h, w, rng, "noise" if rng.integers(3) == 0 else "smooth")
        raw = bytearray(scanlines(s, ctype, depth, inter, lambda r: int(rng.integers(5))))
        cinfo = int(rng.integers(0, 8))
        maxdist = int(rng.integers(1, (1 << (cinfo + 8)) + 1)) if rng.integers(3) else 1 << (cinfo + 8)
        d = Deflate()
        p, nraw = 0, len(raw)
        while True:
            n_b = int(rng.integers(0, max(2, nraw // int(rng.integers(1, 6)))))
            hi = min(nraw, p + n_b)
            final = hi == nraw and rng.integers(4) > 0
            t = int(rng.integers(10))
            if t == 0 and hi - p < 65536:
                d.stored(bytes(raw[p:hi]), final)
            else:
                toks = lz77(raw, p, hi, maxdist=maxdist, maxlen=int(rng.choice([3, 10, 258])),
                            use284=bool(rng.integers(2)))
                if t <= 3:
                    d.fixed(toks, final)
                else:
                    has_d = any(not isinstance(x, int) for x in toks)
                    kw = dict(limit=int(rng.integers(9, 16)), fib=bool(rng.integers(3) == 0),
                              use16=bool(rng.integers(4)), use17=bool(rng.integers(4)), use18=bool(rng.integers(4)),
                              joint=bool(rng.integers(2)), hclen=int(rng.integers(4, 20)),
                              nl=int(rng.integers(257, 287)), nd=int(rng.integers(1, 31)))
                    if not has_d and rng.integers(3) == 0:
                        kw["dist"] = "none" if rng.integers(2) else "one"
                    d.dynamic(toks, final, **kw)
            p = hi
            if final:
                break
        out.append(case("sweep_%03d_t%d_d%d_i%d_%dx%d_w%d" % (i, ctype, depth, inter, h, w, cinfo), d, raw, None,
                        cinfo=cinfo, ctype=ctype, depth=depth, shape=s.shape, interlace=inter))
    return out


def cases(seed=11, n_sweep=300):
    rng = np.random.default_rng(seed)
    out = [_symbol_cap(rng)]
    out += _block_cap(rng)
    out.append(_candidate_flood(rng))
    out += _cross_boundary(rng)
    out += _unusual_codes(rng)
    out.append(_len258(rng))
    out += _window(rng)
    out.append(_alignment(rng))
    out += _both_refuse(rng)
    out += _sweep(rng, n_sweep)
    return out


def adversarial(seed=11, n_sweep=300):
    return [(c.name, c.png, c.expect) for c in cases(seed, n_sweep)]
