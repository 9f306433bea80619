"""CPU restatement of the GPU PNG encoder (smap_b200/csrc/png_enc.cu), pinned byte for byte against
cv2.imencode(".png", bgr) (libpng 1.6 with zlib 1.2.11) and against Python's zlib by tests/test_png_encode_cpu.py.  It never
calls zlib.compress: every stage below is one the kernels compute, so each can be compared with their intermediates.

    s = filtered(bgr)                  # RGB scanlines, filter byte 1 (Sub) per row; filter 0 (None) when W = 1
    syms, pos = parse(s)               # zlib's deflate_rle tokens: literals 0..255, matches 256 + (len - 3), distance 1
    blocks = split(syms, pos, len(s))  # 16383 symbols per block, a final block always (empty after an exact multiple)
    plan = block_plan(...)             # per block: zlib's trees, stored / fixed / dynamic choice, bit size
    z = zlib_stream(s)                 # CMF/FLG (libpng's window rewrite), the packed blocks, Adler-32
    encode(bgr)                        # signature, IHDR, 8192-byte IDAT chunks, IEND

The parse is context free because Z_RLE only looks one byte back: inside a maximal run of equal bytes the first byte is
a literal (or the run starts the stream), then 258-long matches, then one match of 3..257 or 0..2 literals.  The trees
are zlib's trees.c: build_tree with its heap order and depth tie-break and the rule that a tree has at least two codes,
gen_bitlen's overflow repair, scan_tree / send_tree run lengths, the bl_order trim to at least 4 code-length codes, and
_tr_flush_block's choice between stored (only while the block's bytes are still in the window), fixed and dynamic.
"""
import struct
import zlib as _zlib  # crc32 and adler32 only

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
BLOCK_SYMS = 16383  # lit_bufsize - 1 at memLevel 8: zlib flushes a block when this many symbols are tallied
IDAT_BYTES = 8192  # libpng's zbuf size: the zlib stream is cut into chunks of this many bytes
MAX_MATCH, MIN_LOOKAHEAD = 258, 262

# deflate's length codes: base lengths (minus 3) and extra bits of codes 257..285
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
LEN_BASE = []
_b = 0
for _e in LEN_EXTRA[:-1]:
    LEN_BASE.append(_b)
    _b += 1 << _e
LEN_BASE.append(255)
LEN_CODE = np.zeros(256, np.int64)  # match length - 3 -> code - 257
for _c in range(28):
    LEN_CODE[LEN_BASE[_c]:LEN_BASE[_c] + (1 << LEN_EXTRA[_c])] = _c
LEN_CODE[255] = 28
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
BL_EXTRA = [0] * 16 + [2, 3, 7]
STATIC_LLEN = np.array([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, np.int64)  # 288 codes; 286 are used
STATIC_DLEN = np.full(30, 5, np.int64)


# ---- 1. filtered stream ------------------------------------------------------------------------------------------------
def filtered(bgr):
    """uint8 BGR [H, W, 3] -> the scanlines libpng deflates: per row a filter byte, then the RGB bytes; filter 1 (Sub,
    x[i] - x[i-3] mod 256) unless W = 1, where every row is filter 0 (None)."""
    h, w, _ = bgr.shape
    rgb = np.ascontiguousarray(bgr[..., ::-1]).reshape(h, 3 * w)
    f = rgb.copy()
    if w > 1:
        f[:, 3:] = rgb[:, 3:] - rgb[:, :-3]  # uint8 wraps mod 256
    fb = np.full((h, 1), 1 if w > 1 else 0, np.uint8)
    return np.concatenate([fb, f], 1).reshape(-1)


def window_bits(n):
    """zlib windowBits libpng asks for, for n bytes of scanlines."""
    wbits = 15
    if n <= 16384:
        half = 16384
        while n + MIN_LOOKAHEAD <= half:
            half >>= 1
            wbits -= 1
    return wbits


def zlib_header(n):
    """CMF, FLG: deflate's header for window_bits(n) at level 1 (FLEVEL 0), then libpng's optimize_cmf rewrite."""
    cmf = 8 | ((window_bits(n) - 8) << 4)
    if n <= 16384:
        cinfo = cmf >> 4
        half = 1 << (cinfo + 7)
        if n <= half:
            while True:
                half >>= 1
                cinfo -= 1
                if not (cinfo > 0 and n <= half):
                    break
            cmf = (cmf & 15) | (cinfo << 4)
    flg = 31 - (cmf * 256) % 31
    return cmf, flg


# ---- 2. token parse ------------------------------------------------------------------------------------------------
def parse(s):
    """-> (syms, pos): deflate_rle's symbols in order (0..255 a literal, 256 + len - 3 a match of length len at distance
    1) and the stream position each starts at.  Per maximal run of L equal bytes: a literal, then (L - 1) // 258 matches
    of 258, then the rest m = (L - 1) % 258 as one match (m >= 3) or m literals."""
    n = len(s)
    start = np.flatnonzero(np.r_[True, s[1:] != s[:-1]])
    L = np.diff(np.r_[start, n])
    r = L - 1
    q, m = r // 258, r % 258
    tail = np.where(m >= 3, 1, m)
    cnt = 1 + q + tail
    first = np.cumsum(cnt) - cnt  # the run's first symbol
    total = int(cnt.sum())
    run = np.repeat(np.arange(len(start)), cnt)
    k = np.arange(total) - first[run]  # symbol number inside its run
    a = start[run]
    qq, mm = q[run], m[run]
    pos = np.where(k == 0, a, np.where(k <= qq, a + 1 + 258 * (k - 1), a + 1 + 258 * qq + (k - 1 - qq)))
    ln = np.where(k == 0, 1, np.where(k <= qq, 258, np.where(mm >= 3, mm, 1)))
    syms = np.where(ln >= 3, 256 + ln - 3, s[pos].astype(np.int64))
    return syms.astype(np.int64), pos.astype(np.int64)


# ---- 3. block split and the window ---------------------------------------------------------------------------------
def window_offset(p, n, wsize):
    """Bytes slid out of zlib's 2 * wsize window when its loop reaches position p (a symbol's start, or n at the end).
    fill_window runs when at most 258 bytes are left in the window and slides once the position is at or past
    2 * wsize - 262 in it; with the whole input available the window is refilled to its end at each slide, so slide k
    (k >= 1) happens at the first symbol start >= (k + 1) wsize - 258 while (k + 1) wsize < n, and one last slide may
    come within the final 258 bytes at the first start >= max(n - 258, (k + 1) wsize - 262)."""
    ka = max(0, (n - 1) // wsize - 1)  # slides made while the input still reaches past the window
    cnt = min(ka, max(0, (p + MAX_MATCH) // wsize - 1))
    if cnt == ka and p >= max(n - MAX_MATCH, (ka + 2) * wsize - MIN_LOOKAHEAD):
        cnt += 1
    return cnt * wsize


def split(syms, pos, n):
    """-> list of (sym0, sym1, pos0, pos1, flush_pos, last): the blocks' symbol ranges, their byte ranges, and the position
    zlib's loop is at when it flushes the block."""
    nb = len(syms) // BLOCK_SYMS + 1
    out = []
    for b in range(nb):
        s0, s1 = b * BLOCK_SYMS, min(len(syms), (b + 1) * BLOCK_SYMS)
        p0 = int(pos[s0]) if s0 < len(syms) else n
        p1 = int(pos[s1]) if s1 < len(syms) else n
        last = b == nb - 1
        flush = n if last else int(pos[s1 - 1])
        out.append((s0, s1, p0, p1, flush, last))
    return out


# ---- 4. trees (zlib trees.c) ---------------------------------------------------------------------------------------
class Tree:
    """One build_tree: code lengths, codes, max_code, and what it adds to opt_len / static_len."""

    def __init__(self, freq, stree, extra, base, max_length):
        elems = len(freq)
        nodes = 2 * elems + 1
        f = np.zeros(nodes, np.int64)
        f[:elems] = freq
        self.freq = f
        length = np.zeros(nodes, np.int64)
        dad = np.zeros(nodes, np.int64)
        depth = np.zeros(nodes, np.int64)
        heap = [0] * (2 * 286 + 2)
        heap_len, heap_max = 0, 2 * 286 + 1  # HEAP_SIZE = 2 * L_CODES + 1 for every tree (one shared heap in zlib)
        HEAP_SIZE = heap_max
        max_code = -1
        opt = stat = 0
        for i in range(elems):
            if f[i]:
                heap_len += 1
                heap[heap_len] = max_code = i
        while heap_len < 2:  # node = (max_code < 2 ? ++max_code : 0)
            if max_code < 2:
                max_code += 1
                node = max_code
            else:
                node = 0
            heap_len += 1
            heap[heap_len] = node
            f[node] = 1
            depth[node] = 0
            opt -= 1
            if stree is not None:
                stat -= stree[node]

        def smaller(a, b):
            return f[a] < f[b] or (f[a] == f[b] and depth[a] <= depth[b])

        def down(k):
            v = heap[k]
            j = k << 1
            while j <= heap_len:
                if j < heap_len and smaller(heap[j + 1], heap[j]):
                    j += 1
                if smaller(v, heap[j]):
                    break
                heap[k] = heap[j]
                k = j
                j <<= 1
            heap[k] = v

        for k in range(heap_len // 2, 0, -1):
            down(k)
        node = elems
        while True:
            n_ = heap[1]
            heap[1] = heap[heap_len]
            heap_len -= 1
            down(1)
            m_ = heap[1]
            heap_max -= 1
            heap[heap_max] = n_
            heap_max -= 1
            heap[heap_max] = m_
            f[node] = f[n_] + f[m_]
            depth[node] = max(depth[n_], depth[m_]) + 1
            dad[n_] = dad[m_] = node
            heap[1] = node
            node += 1
            down(1)
            if heap_len < 2:
                break
        heap_max -= 1
        heap[heap_max] = heap[1]
        # gen_bitlen
        bl_count = [0] * 16
        length[heap[heap_max]] = 0
        overflow = 0
        h = heap_max + 1
        while h < HEAP_SIZE:
            n_ = heap[h]
            bits = length[dad[n_]] + 1
            if bits > max_length:
                bits, overflow = max_length, overflow + 1
            length[n_] = bits
            h += 1
            if n_ > max_code:
                continue
            bl_count[bits] += 1
            xb = extra[n_ - base] if n_ >= base else 0
            opt += int(f[n_]) * (bits + xb)
            if stree is not None:
                stat += int(f[n_]) * (int(stree[n_]) + xb)
        if overflow:
            while overflow > 0:
                bits = max_length - 1
                while bl_count[bits] == 0:
                    bits -= 1
                bl_count[bits] -= 1
                bl_count[bits + 1] += 2
                bl_count[max_length] -= 1
                overflow -= 2
            for bits in range(max_length, 0, -1):
                c = bl_count[bits]
                while c:
                    h -= 1
                    m_ = heap[h]
                    if m_ > max_code:
                        continue
                    if length[m_] != bits:
                        opt += (bits - int(length[m_])) * int(f[m_])
                        length[m_] = bits
                    c -= 1
        self.len = length[:elems].copy()  # 0 for every symbol outside the heap
        self.max_code, self.opt, self.stat = max_code, opt, stat
        self.code = canonical_codes(self.len)


def canonical_codes(lens):
    """gen_codes: bit-reversed canonical codes (deflate sends them LSB first)."""
    lens = [int(x) for x in lens]
    bl_count = [0] * 16
    for x in lens:
        if x:
            bl_count[x] += 1
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + (bl_count[b - 1] if b > 1 else 0)) << 1
        nxt[b] = code
    out = np.zeros(len(lens), np.int64)
    for i, x in enumerate(lens):
        if x:
            c = nxt[x]
            nxt[x] += 1
            out[i] = int(format(c, "0%db" % x)[::-1], 2)
    return out


def tree_runs(lens, max_code):
    """scan_tree / send_tree: the code-length sequence of lens[0..max_code] as (symbol, extra value, extra bits)."""
    out = []
    prevlen, nextlen, count = -1, int(lens[0]), 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for i in range(max_code + 1):
        curlen = nextlen
        nextlen = int(lens[i + 1]) if i + 1 <= max_code else 0xFFFF
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            out += [(curlen, 0, 0)] * count
        elif curlen != 0:
            if curlen != prevlen:
                out.append((curlen, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


STATIC_LCODE = canonical_codes(STATIC_LLEN)
STATIC_DCODE = canonical_codes(STATIC_DLEN)


def block_plan(bsyms, stored_len, stored_ok):
    """_tr_flush_block for one block's symbols -> dict: type (0 stored, 1 fixed, 2 dynamic), the literal/length and
    distance code lengths and codes it sends with, the dynamic header's pieces and the block's size in bits (stored:
    without the padding to the byte boundary)."""
    lfreq = np.bincount(np.where(bsyms < 256, bsyms, 257 + LEN_CODE[np.clip(bsyms - 256, 0, 255)]), minlength=286)[:286]
    lfreq = lfreq.astype(np.int64)
    lfreq[256] = 1
    nmatch = int((bsyms >= 256).sum())
    dfreq = np.zeros(30, np.int64)
    dfreq[0] = nmatch
    lt = Tree(lfreq, STATIC_LLEN, LEN_EXTRA, 257, 15)
    dt = Tree(dfreq, STATIC_DLEN, [0] * 30, 0, 15)
    runs = tree_runs(lt.len, lt.max_code) + tree_runs(dt.len, dt.max_code)
    blfreq = np.zeros(19, np.int64)
    for sym, _, _ in runs:
        blfreq[sym] += 1
    bt = Tree(blfreq, None, BL_EXTRA, 0, 7)
    max_blindex = 18
    while max_blindex >= 3 and bt.len[BL_ORDER[max_blindex]] == 0:
        max_blindex -= 1
    opt = lt.opt + dt.opt + bt.opt + 3 * (max_blindex + 1) + 14
    stat = lt.stat + dt.stat
    opt_lenb, static_lenb = (opt + 3 + 7) >> 3, (stat + 3 + 7) >> 3
    opt_lenb = min(opt_lenb, static_lenb)
    P = dict(stored_len=stored_len)
    if stored_len + 4 <= opt_lenb and stored_ok:
        P.update(type=0, bits=3 + 32 + 8 * stored_len)
    elif static_lenb == opt_lenb:
        P.update(type=1, bits=stat + 3, llen=STATIC_LLEN[:286], lcode=STATIC_LCODE[:286], dlen=STATIC_DLEN, dcode=STATIC_DCODE)
    else:
        P.update(type=2, bits=opt + 3, llen=lt.len, lcode=lt.code, dlen=dt.len, dcode=dt.code, runs=runs, bllen=bt.len,
                 blcode=bt.code, lcodes=lt.max_code + 1, dcodes=dt.max_code + 1, blcodes=max_blindex + 1)
    return P


def plans(s):
    """The parse, the split and every block's plan of filtered stream s."""
    n = len(s)
    syms, pos = parse(s)
    wsize = 1 << window_bits(n)
    out = []
    for s0, s1, p0, p1, flush, last in split(syms, pos, n):
        P = block_plan(syms[s0:s1], p1 - p0, p0 - window_offset(flush, n, wsize) >= 0)
        P.update(sym0=s0, sym1=s1, pos0=p0, pos1=p1, last=last)
        out.append(P)
    return syms, out


# ---- 5. packing ----------------------------------------------------------------------------------------------------
class BitWriter:
    """LSB-first bit packing; pieces are numpy arrays of (value, length)."""

    def __init__(self):
        self.chunks, self.acc, self.nacc = [], 0, 0

    def bits(self, vals, lens):
        vals = np.asarray(vals, np.int64)
        lens = np.asarray(lens, np.int64)
        keep = lens > 0
        vals, lens = vals[keep], lens[keep]
        if len(lens) == 0:
            return
        total = int(lens.sum())
        own = np.repeat(np.arange(len(lens)), lens)
        bitpos = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
        b = ((vals[own] >> bitpos) & 1).astype(np.uint8)
        if self.nacc:
            b = np.concatenate([((self.acc >> np.arange(self.nacc)) & 1).astype(np.uint8), b])
        whole = len(b) // 8 * 8
        self.chunks.append(np.packbits(b[:whole], bitorder="little").tobytes())
        rest = b[whole:]
        self.acc = int(np.packbits(rest, bitorder="little")[0]) if len(rest) else 0
        self.nacc = len(rest)

    def align(self):
        if self.nacc:
            self.chunks.append(bytes([self.acc]))
        self.acc = self.nacc = 0

    def raw(self, data):
        assert self.nacc == 0
        self.chunks.append(bytes(data))

    def getvalue(self):
        return b"".join(self.chunks) + (bytes([self.acc]) if self.nacc else b"")


def symbol_bits(syms, P):
    """Each symbol's (value, length) under the block's codes: a literal, or a length code, its extra bits and distance 1."""
    lit = syms < 256
    lc = LEN_CODE[np.clip(syms - 256, 0, 255)]
    lsym = np.where(lit, syms, 257 + lc)
    code, ln = P["lcode"][lsym], P["llen"][lsym]
    xb = np.where(lit, 0, np.array(LEN_EXTRA)[lc])
    xv = np.where(lit, 0, syms - 256 - np.array(LEN_BASE)[lc])
    d_c, d_l = int(P["dcode"][0]), int(P["dlen"][0])
    val = code | (xv << ln) | np.where(lit, 0, d_c << (ln + xb))
    return val, ln + xb + np.where(lit, 0, d_l)


def deflate(s):
    """The raw DEFLATE data of filtered stream s, block by block."""
    syms, P_all = plans(s)
    W = BitWriter()
    for P in P_all:
        W.bits([P["type"] << 1 | P["last"]], [3])
        if P["type"] == 0:
            W.align()
            L = P["stored_len"]
            W.raw(struct.pack("<HH", L, L ^ 0xFFFF) + s[P["pos0"]:P["pos1"]].tobytes())
            continue
        if P["type"] == 2:
            hv = [P["lcodes"] - 257, P["dcodes"] - 1, P["blcodes"] - 4] + [int(P["bllen"][BL_ORDER[i]]) for i in range(P["blcodes"])]
            hl = [5, 5, 4] + [3] * P["blcodes"]
            for sym, xv, xb in P["runs"]:
                hv += [int(P["blcode"][sym]), xv]
                hl += [int(P["bllen"][sym]), xb]
            W.bits(hv, hl)
        v, ln = symbol_bits(syms[P["sym0"]:P["sym1"]], P)
        W.bits(np.r_[v, P["lcode"][256]], np.r_[ln, P["llen"][256]])
    W.align()
    return W.getvalue()


def zlib_stream(s):
    cmf, flg = zlib_header(len(s))
    return bytes([cmf, flg]) + deflate(s) + struct.pack(">I", _zlib.adler32(s.tobytes()))


# ---- 6. framing ----------------------------------------------------------------------------------------------------
def chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", _zlib.crc32(kind + data))


def frame_png(h, w, z):
    out = [SIG, chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))]
    out += [chunk(b"IDAT", z[i:i + IDAT_BYTES]) for i in range(0, len(z), IDAT_BYTES)]
    return b"".join(out + [chunk(b"IEND", b"")])


def encode(bgr):
    """uint8 BGR [H, W, 3] -> the bytes cv2.imencode(".png", bgr) writes."""
    h, w, _ = bgr.shape
    return frame_png(h, w, zlib_stream(filtered(bgr)))
