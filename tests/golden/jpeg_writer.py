"""Seeded writer of baseline JPEG files from quantised coefficients, and the files libjpeg never writes that the GPU
decoder must still decode like cv2 (tests/test_jpeg_writer_cpu.py, tests/test_jpeg_writer_gpu.py).

write() codes a coefficient array in the frame-MCU layout of oracle/jpeg_numpy.py (int [nmcu * blocks per MCU, 64],
natural order, absolute DC) as libjpeg does by default, with control over the frame (SOF0 / SOF1, grayscale or the four
samplings), the quantisers (8- or 16-bit DQT, table ids 0-3), the Huffman tables (ids 0-3, several DHT segments, a table
redefined before the SOS, explicit code lengths), the restart interval, per-block token lists that replace libjpeg's
(ZRL + EOB, a ZRL ending at 63, runs past 63), the padding bits, extra entropy bytes and APPn / COM markers before the SOS.
Tokens are coded and packed with numpy, so files of 10^5 dense blocks or 2^16 MCUs take well under a second.

families() lists every file with its expected outcome: "decode" (equal to cv2) or the status the decoder refuses it with
(oracle/jpeg_numpy.py's codes), from smapb_jpeg_info (refused at the header) or from the device decode.

predicted_passes() restates scan_sync_kernel and the host loop that launches it (smap_b200/csrc/jpeg.cu) on the CPU: the
first quiet sync pass of a baseline file at a subsequence length, and the launches one decode of it takes."""
import numpy as np

from jpeg_scans import _codes, _optimal_table
from oracle import jpeg_numpy as J

ZZ = J.ZIGZAG
SAMPLINGS = {"gray": None, "444": (1, 1), "422": (2, 1), "440": (1, 2), "420": (2, 2)}
DECODE = "decode"

# the decoder's constants (smap_b200/csrc/jpeg.cu)
WARM_BITS, PASS_GROUP = 1024, 8
FIXED_LAUNCHES = 6  # unstuff, prefix, write, DC prediction, IDCT, colour


# ---- geometry ----------------------------------------------------------------------------------------------------------
def geometry(h, w, samp):
    """-> dict: comps [(id, h, v)], hmax, vmax, mcux, mcuy, nmcu, lay (component of each block of an MCU)."""
    if samp == "gray":
        comps = [(1, 1, 1)]
    else:
        hs, vs = SAMPLINGS[samp]
        comps = [(1, hs, vs), (2, 1, 1), (3, 1, 1)]
    hmax, vmax = comps[0][1], comps[0][2]
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    lay = [c for c, (_, hs, vs) in enumerate(comps) for _ in range(hs * vs)]
    return dict(h=h, w=w, comps=comps, hmax=hmax, vmax=vmax, mcux=mcux, mcuy=mcuy, nmcu=mcux * mcuy, lay=lay)


def size_for_blocks(samp, blocks, dh=3, dw=5):
    """(h, w) of a frame of about `blocks` blocks whose last MCU row and column are partial."""
    g = geometry(8, 8, samp)
    m = max(1, int(np.ceil(np.sqrt(blocks / len(g["lay"])))))
    return m * 8 * g["vmax"] - dh, m * 8 * g["hmax"] - dw


# ---- tokens ------------------------------------------------------------------------------------------------------------
def _category(v):
    return np.frexp(np.abs(v).astype(np.float64))[1].astype(np.int64)


def _extra(v, s):
    return np.where(v >= 0, v, v + (1 << s) - 1).astype(np.int64)


def tokens(coef, g, dri=0, override=None):
    """libjpeg's token stream of a sequential scan, as arrays in decode order: block, table (2 * component + 0 for DC / 1
    for AC), symbol, extra bits, their count.  override: {block: [("dc" | "ac", symbol, value)]} replaces a block's tokens
    (value: the coefficient the extra bits code; the category is the symbol's low nibble)."""
    coef = np.asarray(coef, np.int64)
    lay = np.asarray(g["lay"])
    bpm = len(lay)
    n = len(coef)
    assert n == g["nmcu"] * bpm, (n, g["nmcu"], bpm)
    comp = np.tile(lay, g["nmcu"])
    seg = np.arange(n) // bpm // (dri or g["nmcu"])
    z = coef[:, ZZ]
    # DC differences, the predictor reset at every restart
    diff = np.empty(n, np.int64)
    for c in range(lay.max() + 1):
        idx = np.flatnonzero(comp == c)
        v = z[idx, 0]
        prev = np.concatenate([[0], v[:-1]])
        prev[np.concatenate([[True], seg[idx][1:] != seg[idx][:-1]])] = 0
        diff[idx] = v - prev
    s_dc = _category(diff)
    blk = [np.arange(n)]
    seq = [np.zeros(n, np.int64)]
    tab = [2 * comp]
    sym = [s_dc]
    val = [_extra(diff, s_dc)]
    nb = [s_dc]
    # AC: runs of zeros, ZRLs for runs of 16 and more, EOB after the last nonzero coefficient unless it is 63
    b, k = np.nonzero(z[:, 1:])
    k = k + 1
    first = np.concatenate([[True], b[1:] != b[:-1]])
    prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prevk - 1
    v = z[b, k]
    s = _category(v)
    nzrl = run // 16
    for j in range(3):
        m = nzrl > j
        blk.append(b[m]), seq.append(4 * k[m] + j), tab.append(2 * comp[b[m]] + 1), sym.append(np.full(m.sum(), 0xF0))
        val.append(np.zeros(m.sum(), np.int64)), nb.append(np.zeros(m.sum(), np.int64))
    blk.append(b), seq.append(4 * k + 3), tab.append(2 * comp[b] + 1), sym.append(((run % 16) << 4) | s)
    val.append(_extra(v, s)), nb.append(s)
    last = np.zeros(n, np.int64)
    last[b] = k  # k ascends within a block: the last assignment wins
    e = np.flatnonzero(last < 63)
    blk.append(e), seq.append(np.full(len(e), 4 * 64)), tab.append(2 * comp[e] + 1), sym.append(np.zeros(len(e), np.int64))
    val.append(np.zeros(len(e), np.int64)), nb.append(np.zeros(len(e), np.int64))
    T = [np.concatenate(a).astype(np.int64) for a in (blk, seq, tab, sym, val, nb)]
    if override:
        keep = ~np.isin(T[0], list(override))
        T = [a[keep] for a in T]
        extra = [[], [], [], [], [], []]
        for bi, toks in override.items():
            for j, (cls, sy, x) in enumerate(toks):
                ss = sy & 15
                for a, y in zip(extra, (bi, j, 2 * lay[bi % bpm] + (cls == "ac"), sy, int(_extra(np.int64(x), ss)), ss)):
                    a.append(y)
        T = [np.concatenate([a, np.asarray(x, np.int64)]) for a, x in zip(T, extra)]
    order = np.lexsort((T[1], T[0]))
    return [a[order] for a in T]


# ---- Huffman tables ----------------------------------------------------------------------------------------------------
def table_from_lengths(lengths):
    """{symbol: code length} -> (counts[16], symbols) in canonical order (by length, then as given)."""
    syms = sorted(lengths, key=lambda s: lengths[s])
    counts = [0] * 16
    for s in syms:
        counts[lengths[s] - 1] += 1
    return counts, syms


def _lut(counts, syms):
    code, ln = np.zeros(256, np.int64), np.zeros(256, np.int64)
    for s, (c, n) in _codes(counts, syms).items():
        if ln[s] == 0:  # a symbol listed twice: the writer uses its first code
            code[s], ln[s] = c, n
    return code, ln


# ---- bit packing -------------------------------------------------------------------------------------------------------
def pack(vals, lens):
    """Concatenates codes (vals[i] in lens[i] <= 32 bits, MSB first) -> (bytes, bit count)."""
    vals = np.asarray(vals, np.uint64)
    lens = np.asarray(lens, np.int64)
    if len(lens) == 0:
        return b"", 0
    off = np.cumsum(lens) - lens
    total = int(off[-1] + lens[-1])
    words = np.zeros(total // 64 + 2, np.uint64)
    w, end = off >> 6, (off & 63) + lens
    fit = end <= 64
    lo = np.where(fit, vals << np.clip(64 - end, 0, 63).astype(np.uint64), vals >> np.clip(end - 64, 0, 63).astype(np.uint64))
    np.bitwise_or.at(words, w, lo)
    sp = ~fit
    np.bitwise_or.at(words, w[sp] + 1, vals[sp] << (128 - end[sp]).astype(np.uint64))
    return words.byteswap().tobytes()[:(total + 7) // 8], total


def stuff(b):
    a = np.frombuffer(bytes(b), np.uint8)
    return np.insert(a, np.flatnonzero(a == 0xFF) + 1, 0).tobytes()


PADS = {"ones": 0xFF, "zeros": 0x00, "mixed": 0x5A}


def _segment(code, ln, pad):
    data, nbits = pack(code, ln)
    k = -nbits % 8
    if k:
        data = data[:-1] + bytes([data[-1] | (PADS[pad] & ((1 << k) - 1))])
    return data


# ---- the file ----------------------------------------------------------------------------------------------------------
def _marker(m, body):
    return bytes([0xFF, m]) + (len(body) + 2).to_bytes(2, "big") + bytes(body)


def write(coef, h, w, samp="420", q=1, qbits=None, qids=None, hids=None, lengths=None, sof=0xC0, dri=0, override=None,
          pad="ones", seg_extra=b"", tail_extra=b"", markers=(), split_dht=False, decoy=False, jfif=True):
    """-> a baseline JPEG file.  q: one quantiser for every component (int or 64 values, natural order) or a list of one
    per component; qids: DQT id of each component (default 0, 1, 1); hids: (DC id, AC id) of each component (default
    (0, 0), (1, 1), (1, 1)); lengths: {(class, component): {symbol: length}} for explicit codes, else libjpeg's optimal
    table from the symbol counts; seg_extra: entropy-coded bytes appended to every restart segment but the last,
    tail_extra: after the last MCU (both stuffed); markers: raw marker segments between the DHT and the SOS; split_dht:
    one DHT segment per table; decoy: define every AC table once more with other codes first (the later one wins)."""
    g = geometry(h, w, samp)
    nc = len(g["comps"])
    qs = q if isinstance(q, list) and len(q) == nc and np.ndim(q[0]) else [q] * nc
    qs = [np.broadcast_to(np.asarray(x, np.int64), (64,)) for x in qs]
    qids = qids or [0, 1, 1][:nc]
    hids = hids or [(0, 0), (1, 1), (1, 1)][:nc]
    lengths = lengths or {}
    blk, _, tab, sym, val, nb = tokens(coef, g, dri, override)
    # tables: one per (class, component), shared when two components use the same id
    luts, dht = {}, []
    for c in range(nc):
        for cls in (0, 1):
            tid = hids[c][cls]
            if (cls, tid) in luts:
                continue
            if (cls, c) in lengths:
                counts, syms = table_from_lengths(lengths[(cls, c)])
            else:
                users = [2 * e + cls for e in range(nc) if hids[e][cls] == tid]
                freq = np.bincount(sym[np.isin(tab, users)], minlength=256)
                counts, syms = _optimal_table([int(x) for x in freq])
            luts[(cls, tid)] = _lut(counts, syms)
            dht.append(bytes([(cls << 4) | tid]) + bytes(counts) + bytes(syms))
    code = np.empty(len(sym), np.int64)
    ln = np.empty(len(sym), np.int64)
    for c in range(nc):
        for cls in (0, 1):
            m = tab == 2 * c + cls
            cd, l = luts[(cls, hids[c][cls])]
            assert (l[sym[m]] > 0).all(), "symbol without a code in table %s" % ((cls, c),)
            code[m], ln[m] = cd[sym[m]], l[sym[m]]
    vals = (code << nb) | val
    lens = ln + nb
    out = bytearray(b"\xff\xd8")
    if jfif:
        out += _marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in sorted(set(qids)):
        qv = qs[qids.index(t)][ZZ]
        if (qbits or (16 if qv.max() > 255 else 8)) == 16:
            out += _marker(0xDB, bytes([0x10 | t]) + qv.astype(">u2").tobytes())
        else:
            out += _marker(0xDB, bytes([t]) + qv.astype(np.uint8).tobytes())
    body = bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc])
    for c, (cid, hs, vs) in enumerate(g["comps"]):
        body += bytes([cid, (hs << 4) | vs, qids[c]])
    out += _marker(sof, body)
    if decoy:
        for t in dht:
            if t[0] >> 4:
                out += _marker(0xC4, bytes([t[0]]) + bytes([0, 2] + [0] * 14) + b"\x00\x01")
    if split_dht:
        for t in dht:
            out += _marker(0xC4, t)
    else:
        out += _marker(0xC4, b"".join(dht))
    if dri:
        out += _marker(0xDD, dri.to_bytes(2, "big"))
    for m in markers:
        out += m
    sos = bytes([nc]) + b"".join(bytes([cid, (hids[c][0] << 4) | hids[c][1]]) for c, (cid, _, _) in enumerate(g["comps"]))
    out += _marker(0xDA, sos + bytes([0, 63, 0]))
    seg_of = blk // len(g["lay"]) // (dri or g["nmcu"])
    nseg = -(-g["nmcu"] // dri) if dri else 1
    cuts = np.searchsorted(seg_of, np.arange(nseg + 1))
    for s in range(nseg):
        a, b = cuts[s], cuts[s + 1]
        data = _segment(vals[a:b], lens[a:b], pad) + (seg_extra if s < nseg - 1 else tail_extra)
        out += stuff(data)
        if s < nseg - 1:
            out += bytes([0xFF, 0xD0 + s % 8])
    return bytes(out + b"\xff\xd9")


# ---- coefficients ------------------------------------------------------------------------------------------------------
def pass1(coef, q):
    """Dequantised coefficients and pass-1 outputs of the decoder's IDCT: -> (max |dequantised|, max |pass 1|) per block."""
    c = np.asarray(coef, np.int64).reshape(-1, 8, 8) * np.asarray(q, np.int64).reshape(8, 8)
    p = np.stack(J._idct_1d(*[c[:, k, :] for k in range(8)], 11), axis=1)
    return np.abs(c).reshape(len(c), -1).max(1), np.abs(p).reshape(len(p), -1).max(1)


def dense_blocks(rng, n, q, dc_max=1023):
    """n blocks with all 64 coefficients nonzero, as large as the IDCT guard allows: every dequantised value and every
    pass-1 output within +-GUARD (checked exactly), most blocks within 10 % of it, DC within +-dc_max (DC differences
    stay in categories <= 11)."""
    q = np.asarray(q, np.int64)
    y = rng.standard_normal((n, 64)) * rng.uniform(0.3, 3, (n, 1)) ** rng.integers(0, 2, (n, 1))
    sign = np.where(y >= 0, 1, -1)
    _, p = pass1(np.rint(y * 1000 / q).astype(np.int64), q)  # pass 1 is linear up to rounding: scale towards the guard
    scale = 1000 * J.GUARD * rng.uniform(0.9, 1.0, n) / np.maximum(p, 1)
    c = np.rint(y * scale[:, None] / q).astype(np.int64)
    for _ in range(200):
        c = np.where(c == 0, sign, c)
        c[:, 0] = np.clip(c[:, 0], -dc_max, dc_max)
        dq, p = pass1(c, q)
        bad = (dq > J.GUARD) | (p > J.GUARD)
        if not bad.any():
            return c
        c[bad] = np.trunc(c[bad] * 0.97).astype(np.int64)
    raise AssertionError("dense blocks did not fit the guard")


def dc_blocks(dc, n):
    c = np.zeros((n, 64), np.int64)
    c[:, 0] = dc
    return c


def flat_dc(level):
    """DC coefficient (q = 1) of a block whose pixels all equal `level`: the IDCT gives 128 + DC / 8."""
    return 8 * (np.asarray(level, np.int64) - 128)


# ---- CPU restatement of the sync schedule ------------------------------------------------------------------------------
class _Scan:
    """A baseline file's entropy-coded data as the device sees it: restart segments unstuffed and concatenated."""

    def __init__(self, data):
        hd = J.parse(data)
        d = bytes(data)
        self.lay = J.mcu_layout(hd)
        self.dc = [J._huff_table(*t) for t in hd["dc"]]
        self.ac = [J._huff_table(*t) for t in hd["ac"]]
        buf, self.segs = b"", []
        for a, b in hd["segments"]:
            u = d[a:b].replace(b"\xff\x00", b"\xff")
            self.segs.append((len(buf) * 8, (len(buf) + len(u)) * 8))
            buf += u
        self.buf = buf + b"\x00" * 16

    def run(self, pos, blk, zz, stop, seg_end):
        """scan_run<false>: decodes from (pos, blk, zz) while pos < stop -> (pos, blk, zz)."""
        buf, lay, bpm = self.buf, self.lay, len(self.lay)
        while pos < stop:
            lut = self.dc[lay[blk]] if zz == 0 else self.ac[lay[blk]]
            i = pos >> 3
            e = lut[((int.from_bytes(buf[i:i + 4], "big") << (pos & 7)) >> 16) & 0xFFFF]
            if e == 0:  # not a code: skip one bit
                pos += 1
                continue
            ln, sym = e >> 8, e & 255
            s, r = sym & 15, sym >> 4
            if pos + ln + s > seg_end:
                pos = seg_end
                break
            done = False
            if zz == 0:
                zz = 1
            elif s == 0:
                if r == 15:
                    zz += 16
                    done = zz >= 64
                else:
                    done = True
            else:
                zz += r
                done = zz > 63 or zz + 1 > 63
                zz += 1
            pos += ln + s
            if done:
                zz = 0
                blk = (blk + 1) % bpm
        return pos, blk, zz


def predicted_passes(data, sub_bits=512):
    """-> dict for one baseline file decoded alone at SMAPB_JPEG_SUB_BITS = sub_bits:
    first_quiet  the first sync pass in which no subsequence changes (the passes are 0..first_quiet),
    bound        the latest first_quiet the schedule allows: the subsequences that the 1024-bit warm-up reaches from their
                 segment's start begin exact, and each later pass makes at least one more subsequence exact,
    worst        first_quiet == bound (no guessed subsequence fell into step before its predecessor was exact),
    passes       sync launches the host loop issues (groups of PASS_GROUP, capped at max_nsub_seg + 2),
    launches     every launch of the decode (smapb_launch_count), nsub_seg: subsequences per segment."""
    S = _Scan(data)
    subs = []  # (begin, end, segment begin, segment end, first of its segment)
    nsub_seg = []
    for a, b in S.segs:
        n = max(1, -(-(b - a) // sub_bits))
        nsub_seg.append(n)
        for u in range(n):
            subs.append((min(b, a + u * sub_bits), b if u == n - 1 else a + (u + 1) * sub_bits, a, b, u == 0))
    st = []
    for beg, end, sa, sb, first in subs:  # pass 0: the guess, after a warm-up
        if first:
            start = (beg, 0, 0)
        else:
            fr = beg - min(beg - sa, WARM_BITS)
            start = S.run(fr, 0, 0, beg, sb)
        st.append((start, S.run(*start, end, sb)))
    p = 0
    while True:
        p += 1
        nxt, changed = [], False
        for i, (beg, end, sa, sb, first) in enumerate(subs):
            if first or st[i - 1][1] == st[i][0]:
                nxt.append(st[i])
            else:
                start = st[i - 1][1]
                nxt.append((start, S.run(*start, end, sb)))
                changed = True
        st = nxt
        if not changed:
            break
        assert p <= max(nsub_seg) + 1, "sync passes do not converge"
    warm = WARM_BITS // sub_bits + 1  # subsequences whose warm-up starts at their segment's first bit
    bound = max(max(1, n - warm + 1) for n in nsub_seg)
    assert p <= bound, (p, bound)
    # the host loop: groups of PASS_GROUP launches, then a look at their `changed` flags
    round_passes = max(nsub_seg) + 1
    launched = 0
    while True:
        first, launched = launched, min(launched + PASS_GROUP, round_passes + 1)
        if first <= p < launched:
            break
        assert launched <= round_passes, "did not converge"
    return dict(first_quiet=p, bound=bound, worst=p == bound, passes=launched, launches=launched + FIXED_LAUNCHES,
                nsub_seg=nsub_seg)


# ---- corpus families ---------------------------------------------------------------------------------------------------
def _entry(name, data, expect, coef=None):
    return dict(name=name, data=data, expect=expect, coef=coef)


def dense(seed=31, blocks=4000):
    """Dense random blocks at q = 1, 2, 3, 8 and mixed tables, in the five samplings, frames ending in partial MCUs."""
    rng = np.random.default_rng(seed)
    out = []
    for samp in SAMPLINGS:
        h, w = size_for_blocks(samp, blocks)
        g = geometry(h, w, samp)
        nc = len(g["comps"])
        for qn in (1, 2, 3, 8, "mixed"):
            if qn == "mixed":
                q = [rng.integers(1, 17, 64) for _ in range(nc)]
                qids = list(range(nc))
                qbits = 16 if samp in ("444", "gray") else 8
            else:
                q, qids, qbits = [np.full(64, qn)] * nc, None, None
            coef = np.zeros((g["nmcu"] * len(g["lay"]), 64), np.int64)
            comp = np.tile(g["lay"], g["nmcu"])
            for c in range(nc):
                m = comp == c
                coef[m] = dense_blocks(rng, int(m.sum()), q[c])
            out.append(_entry("dense_%s_q%s_%dx%d" % (samp, qn, w, h), write(coef, h, w, samp, q, qbits=qbits, qids=qids),
                              DECODE, coef))
    return out


def guard_search():
    """Two-coefficient blocks (DC and the coefficient below it, q = 1) whose largest pass-1 output is exactly GUARD and
    GUARD + 1, found with the oracle's IDCT: -> {8191: coef, 8192: coef}."""
    found = {}
    for dc in range(2047, 1900, -1):
        for x in range(-40, 41):
            c = np.zeros((1, 64), np.int64)
            c[0, 0], c[0, 16] = dc, x
            m = int(pass1(c, np.ones(64))[1][0])
            if m in (J.GUARD, J.GUARD + 1) and m not in found:
                found[m] = c[0]
        if len(found) == 2:
            return found
    raise AssertionError("no guard-edge block")


def guard_edges():
    """Blocks at the guard: the largest pass-1 output exactly 8191 (decodes) and 8192 (refused); DC-only blocks whose
    dequantised value is 2047 (pass 1 = 8188, decodes) and 2048 (8192, refused).  A dequantised value beyond 2047 always
    gives a pass-1 output beyond 8191 (pass 1 keeps at least 4x the column's largest input), so 8191 / 8192 on the
    dequantised values themselves cannot be reached."""
    out = []
    rng = np.random.default_rng(33)
    found = guard_search()
    for samp in ("gray", "420"):
        h, w = 13, 21
        g = geometry(h, w, samp)
        n = g["nmcu"] * len(g["lay"])
        base = dense_blocks(rng, n, np.ones(64)) // 4
        for m, expect in ((J.GUARD, DECODE), (J.GUARD + 1, J.UNSUPPORTED)):
            coef = base.copy()
            coef[n // 2] = found[m]
            out.append(_entry("guard_pass1_%d_%s" % (m, samp), write(coef, h, w, samp, 1), expect, coef))
        for dc, expect in ((2047, DECODE), (2048, J.UNSUPPORTED)):
            coef = np.zeros((n, 64), np.int64)
            coef[:, 0] = rng.integers(-2047, 2048, n)
            coef[n - 1, 0] = dc
            out.append(_entry("guard_dc_%d_%s" % (dc, samp), write(coef, h, w, samp, 1), expect, coef))
        coef = base.copy()  # q = 2: the same pass-1 output from half the coefficient
        coef[n // 2] = 0
        coef[n // 2, 0] = 1024
        out.append(_entry("guard_dc_q2_2048_%s" % samp, write(coef, h, w, samp, 2), J.UNSUPPORTED, coef))
    return out


LUMA_LEVELS = np.rint(np.linspace(0, 255, 16)).astype(int)


def colour_file(level):
    """A 2048x2048 4:4:4 file of flat blocks (DC only, q = 1): luma `level` everywhere, one (Cb, Cr) pair per MCU, every
    pair once."""
    cb, cr = np.divmod(np.arange(65536), 256)
    coef = np.zeros((3 * 65536, 64), np.int64)
    coef[0::3, 0] = flat_dc(level)
    coef[1::3, 0] = flat_dc(cb)
    coef[2::3, 0] = flat_dc(cr)
    return _entry("colour_y%d" % level, write(coef, 2048, 2048, "444", 1), DECODE, coef)


def upsampling(seed=35):
    """4:2:0, 4:2:2 and 4:4:0 frames with chroma planes 1 to 4 wide and high (odd and even luma sizes) and at odd sizes
    of several MCUs; dense chroma saturates most chroma pixels, so neighbours are 0 and 255."""
    rng = np.random.default_rng(seed)
    out = []
    sizes = [(h, w) for h in range(1, 9) for w in range(1, 9)] + [(17, 23), (31, 9), (9, 33), (45, 47)]
    for samp in ("420", "422", "440"):
        for h, w in sizes:
            g = geometry(h, w, samp)
            n = g["nmcu"] * len(g["lay"])
            coef = dense_blocks(rng, n, np.full(64, 2))
            out.append(_entry("up_%s_%dx%d" % (samp, w, h), write(coef, h, w, samp, 2), DECODE, coef))
    return out


def _ac_symbols():
    return [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]


def _sparse(rng, n, cats_dc=12, cats_ac=10):
    """Blocks with a DC and a few AC coefficients in row 0 (pass 1 stays 4x the largest), every category at its
    extremes (+-2^(s-1), +-(2^s - 1))."""
    coef = np.zeros((n, 64), np.int64)
    ext = lambda s: [x * sg for x in (1 << (s - 1), (1 << s) - 1) for sg in (1, -1)]  # noqa: E731
    dcs = [0] + [v for s in range(1, cats_dc) for v in ext(s)]
    d = np.array([dcs[i % len(dcs)] for i in range(n)])
    coef[:, 0] = np.where(np.arange(n) % 2, 0, d)  # DC alternates with 0: every difference is one of the extremes
    acs = [v for s in range(1, cats_ac + 1) for v in ext(s)]
    row0 = [1, 2, 3, 4, 5, 6, 7]
    for i in range(n):
        for j in rng.choice(row0, int(rng.integers(0, 4)), replace=False):
            coef[i, j] = acs[int(rng.integers(len(acs)))]
    return coef


def dconly_of(coef):
    c = np.array(coef)
    c[:, 1:] = 0
    return c


def _few_symbols(rng, n):
    """Blocks that use 15 AC value symbols: +-1 after runs of 0..10, +-2..3 after runs of 0..2, +-4..7 right away,
    and EOB (DC as _sparse)."""
    coef = _sparse(rng, n)
    coef[:, 1:] = 0
    coef[:, 0] = np.clip(coef[:, 0], -1900, 1900)  # room for the AC coefficients below the DC in pass 1
    for i in range(n):
        k = 1
        while k < 64 and rng.random() < 0.85:
            s = int(rng.choice([1, 1, 1, 2, 3]))
            r = int(rng.integers(0, {1: 11, 2: 3, 3: 1}[s]))
            if k + r > 63:
                break
            coef[i, ZZ[k + r]] = int(rng.integers(1 << (s - 1), 1 << s)) * int(rng.choice([1, -1]))
            k += r + 1
    return coef


def huffman_edges(seed=37):
    """Files with explicit codes and token streams libjpeg never writes, and the ones among them cv2 reads but the
    decoder refuses."""
    rng = np.random.default_rng(seed)
    out = []
    h, w = 27, 45
    g = geometry(h, w, "420")
    n = g["nmcu"] * len(g["lay"])
    coef = _sparse(rng, n)
    acs = _ac_symbols()
    dcs = list(range(12))

    def add(name, expect=DECODE, c=coef, hh=h, ww=w, samp="420", **kw):
        out.append(_entry(name, write(c, hh, ww, samp, kw.pop("q", 1), **kw), expect, c if "override" not in kw else None))

    # every length 1..16 in the AC code, one code each, the most frequent symbol on the 16-bit code; the blocks use 15
    # value symbols and EOB.  A 17th symbol would take the all-ones word: libjpeg refuses such a table (and every
    # complete code), and so does the decoder
    few = _few_symbols(rng, n)
    T = tokens(few, g)
    freq = np.bincount(T[3][T[2] % 2 == 1], minlength=256)
    by_freq = [int(x) for x in np.argsort(-freq, kind="stable") if freq[x]]
    assert len(by_freq) == 16, by_freq
    lens_ac = {by_freq[0]: 16}
    lens_ac.update({x: i + 1 for i, x in enumerate(by_freq[1:])})
    fdc = np.bincount(T[3][T[2] % 2 == 0], minlength=16)
    dc_by = [int(x) for x in np.argsort(-fdc, kind="stable")[:12]]
    lens_dc = {dc_by[0]: 16}
    lens_dc.update({x: i + 1 for i, x in enumerate(dc_by[1:])})
    L = {(0, 0): lens_dc, (1, 0): lens_ac, (0, 1): lens_dc, (1, 1): lens_ac}
    add("huff_all_lengths", c=few, lengths=L)
    add("huff_all_lengths_rst", c=few, lengths=L, dri=4, pad="zeros")
    full = dict(lens_ac)
    full[0xF0] = 16  # complete: the ZRL (never used) on the all-ones word
    assert sum(2.0 ** -x for x in full.values()) == 1.0
    add("huff_all_ones_ac", J.MALFORMED, c=few, lengths={(0, 0): lens_dc, (1, 0): full, (0, 1): lens_dc, (1, 1): lens_ac})
    add("huff_complete_dc", J.MALFORMED, c=dconly_of(few), lengths={(0, 0): {x: 4 for x in range(16)}, (0, 1): {x: 4 for x in range(16)}})
    # nearly every code at 9 or 10 bits (the split between the decoder's fast table and its maxcode loop), the EOB and
    # DC category 11 at 16 bits
    lens_ac2 = {0x00: 16}
    for i, x in enumerate([x for x in acs if x != 0x00]):
        lens_ac2[x] = 9 if i % 2 else 10
    lens_dc2 = {x: (9 if x % 2 else 10) for x in dcs}
    lens_dc2[11] = 16
    L2 = {(0, 0): lens_dc2, (1, 0): lens_ac2, (0, 1): lens_dc2, (1, 1): lens_ac2}
    add("huff_codes_9_10", lengths=L2)
    add("huff_codes_9_10_gray", hh=8, ww=8 * n, samp="gray",
        lengths={k: v for k, v in L2.items() if k[1] == 0})
    # an AC table with only EOB, on a DC-only image
    add("huff_ac_eob_only", c=dconly_of(coef), lengths={(1, 0): {0x00: 1}, (1, 1): {0x00: 1}})
    # per-component tables with ids 0..3 in several DHT segments, one redefined before the SOS; quantisers with ids 0..3
    # and 16-bit entries of 0, 1 and 32767 where the coefficient is 0
    q0 = np.ones(64, np.int64)
    q0[63] = 32767
    q0[62] = 0
    q1 = rng.integers(1, 4, 64)
    q1[:8] = 1  # row 0 holds the large coefficients
    q1[63] = 32767
    for samp, qids, hids in (("420", [3, 2, 1], [(2, 3), (3, 1), (0, 0)]), ("444", [0, 3, 3], [(1, 2), (1, 2), (3, 3)])):
        gg = geometry(h, w, samp)
        c = _sparse(rng, gg["nmcu"] * len(gg["lay"]))
        c[:, 62] = rng.integers(-5, 6, len(c))  # multiplied by 0 in luma
        add("tables_ids_%s" % samp, c=c, samp=samp, q=[q0, q1, q1], qids=qids, hids=hids, split_dht=True, decoy=True,
            qbits=16)
    add("sof1_app_com", sof=0xC1, markers=[_marker(0xE5, b"app5 payload"), _marker(0xFE, b"a comment"), _marker(0xED, b"")])
    # restart intervals: every MCU, a short last segment, larger than the MCU count; each padding kind; extra bytes at the
    # end of every restart segment and after the last MCU (libjpeg skips them)
    for dri in (1, 7, 10000):
        for pad in ("ones", "zeros", "mixed"):
            add("dri%d_pad_%s" % (dri, pad), dri=dri, pad=pad)
    add("extra_bytes_rst", dri=3, seg_extra=b"\x12\xff\x34\x00", tail_extra=b"\xff\xff\xab")
    add("extra_bytes_tail", tail_extra=bytes(range(256)))
    # token patterns libjpeg never writes
    lone = np.zeros((n, 64), np.int64)
    lone[:, 0] = coef[:, 0]
    lone[:, ZZ[10]] = 5
    ov = {}
    for b in range(0, n, 3):  # ZRL + EOB
        ov[b] = [("dc", 0, 0), ("ac", 0x93, 5), ("ac", 0xF0, 0), ("ac", 0x00, 0)]
    for b in range(1, n, 3):  # a ZRL that ends exactly at 63: no EOB
        ov[b] = [("dc", 0, 0), ("ac", 0x93, 5), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0x43, 5), ("ac", 0xF0, 0)]
    for b in range(2, n, 3):  # the last coefficient at 63 after three ZRLs, no EOB
        ov[b] = [("dc", 0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xE3, -7)]
    ov[0] = [("dc", 11, 1500), ("ac", 0xF0, 0), ("ac", 0x00, 0)]
    ov[3] = [("dc", 11, -1500), ("ac", 0x00, 0)]
    add("tokens_zrl_eob", c=lone, override=ov)
    add("tokens_zrl_eob_rst", c=lone, override=ov, dri=2, pad="zeros")
    bad = {7: [("dc", 0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0x00, 0)]}
    add("tokens_zrl_past_63", J.CORRUPT, c=lone, override=bad)
    bad = {5: [("dc", 0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xF0, 0), ("ac", 0xF1, 1)]}
    add("tokens_run_past_63", J.CORRUPT, c=lone, override=bad)
    # no DHT (Motion-JPEG frames): cv2 decodes them with the standard tables, the decoder leaves them to cv2
    b = write(coef, h, w, "420", 1)
    p = b.find(b"\xff\xc4")
    L = (b[p + 2] << 8) | b[p + 3]
    out.append(_entry("no_dht", b[:p] + b[p + 2 + L:], J.UNSUPPORTED))
    return out


def _alternating(s):
    """The value of category s whose extra bits alternate 1010... (its negation codes 0101...)."""
    return int(("10" * 8)[:s], 2)


def _adversary(L, n_sub, sub_bits, nseg, seed):
    """A grayscale file whose every unit is L bits (L odd): 4-bit DC and AC codes whose symbols all have category
    s = L - 4, the same run pattern in every block, no EOB.  The codes used contain no "11" and the extra bits alternate,
    so no four consecutive bits of the stream are ones: 1111, the one 4-bit word that is not a code (libjpeg refuses a
    code of all ones), never occurs, a decoder that starts at a wrong bit keeps its wrong phase mod L, and one that starts
    at the right bit but the wrong zig-zag index keeps decoding true units.  Each of the `nseg` restart segments is
    padded with zero bytes to exactly n_sub subsequences."""
    rng = np.random.default_rng(seed)
    s = L - 4
    runs = []
    k = 1
    while k < 64:  # zero runs of 1..4, the last coefficient at 63
        r = min(int(rng.integers(1, 5)), 63 - k)
        runs.append(r)
        k += r + 1
    ubits = (1 + len(runs)) * L
    seg_bytes = n_sub * sub_bits // 8
    per = (seg_bytes * 8 - 7) // ubits
    assert per >= 1, (L, n_sub, sub_bits)
    n = per * nseg
    v = _alternating(s)
    coef = np.zeros((n, 64), np.int64)
    coef[:, 0] = np.where(np.arange(n) % per % 2, 0, v)  # every DC difference is +-v, restarts included
    k = 1
    for r in runs:
        k += r
        coef[:, ZZ[k]] = rng.choice([v, -v], n)
        k += 1
    # AC codes 0000, 0001, 0010, 0100, 0101 for runs 0..4; 15 codes in all, 1111 left out
    ac_syms = [0, 1, 2, 5, 3, 4] + list(range(6, 15))
    ac = {(r << 4) | s: 4 for r in ac_syms}
    dc = {s: 4}  # 15 four-bit codes, the first (0000) for category s; the others become s below
    dc.update({x: 4 for x in range(15) if x != s})
    b = write(coef, 8, 8 * n, "gray", 1, lengths={(0, 0): dc, (1, 0): ac}, dri=per if nseg > 1 else 0, pad="zeros")
    hd = J.parse(b)
    p0 = hd["segments"][0][0]
    head = bytearray(b[:p0])
    t = head.find(b"\xff\xc4") + 4
    assert head[t] == 0x00 and head[t + 4] == 15 and head[t + 17] == s
    head[t + 17:t + 32] = bytes([s] * 15)  # every DC code decodes to category s
    body = bytearray()
    for j, (a, e) in enumerate(hd["segments"]):
        seg = b[a:e]
        un = len(seg.replace(b"\xff\x00", b"\xff"))
        assert un <= seg_bytes
        body += seg + bytes(seg_bytes - un)
        if j < len(hd["segments"]) - 1:
            body += bytes([0xFF, 0xD0 + j % 8])
    return bytes(head) + bytes(body) + b"\xff\xd9", coef


SUB_BITS = (32, 64, 512)


def long_units(cat, n=24, dri=5, seed=45):
    """A grayscale file whose units are 16-bit codes plus `cat` extra bits: AC category 10 (26-bit units) or DC category
    11..15 (27 to 31 bits; 12..15 put the DC beyond the guard).  Shorter codes go to symbols the file never uses."""
    rng = np.random.default_rng(seed + cat)
    coef = np.zeros((n, 64), np.int64)
    if cat == 10:
        coef[:, 1:4] = rng.choice([512, -512, 1023, -1023], (n, 3))  # row 0: pass 1 = 4x, within the guard
    else:
        coef[:, 0] = np.where(np.arange(n) % dri % 2, 0, 1 << (cat - 1))
    dc = {x: x for x in range(1, 10)}
    dc.update({0: 16, cat: 16})
    ac = {(x << 4) | 1: x + 1 for x in range(9)}
    ac.update({0x0A: 16, 0x3A: 16, 0x00: 16})
    return write(coef, 8, 8 * n, "gray", 1, lengths={(0, 0): dc, (1, 0): ac}, dri=dri), coef


def sync_adversaries():
    """Files for the sync passes at each subsequence length: segments of exactly 1, 8, 9 and 16 subsequences, the
    lengths at which the passes cross a group of 8 (warm-up reach + 7 and + 8), and longer ones; plus files of 26- and
    27-bit units at 32-bit subsequences (16-bit codes, 10 and 11 extra bits) and their 28- to 31-bit counterparts (DC
    categories 12-15, beyond the guard: decoded, then refused).  -> entries with the `sub_bits` they were made for."""
    out = []
    seed = 40
    dc1 = dc_blocks(np.where(np.arange(40) % 2, 0, 300), 40)
    for sb in SUB_BITS:  # one block per restart segment: one subsequence each
        e = _entry("sync_sub%d_n1" % sb, write(dc1, 8, 8 * 40, "gray", 1, dri=1), DECODE, dc1)
        e["sub_bits"] = sb
        out.append(e)
    for sb in SUB_BITS:
        warm = WARM_BITS // sb + 1
        for n_sub, nseg in ((8, 2), (9, 2), (16, 1), (warm + 7, 2), (warm + 8, 1), (warm + 15, 2)):
            L = (7, 9, 11)[seed % 3]
            data, coef = _adversary(L, n_sub, sb, nseg, seed)
            seed += 1
            e = _entry("sync_sub%d_n%d_L%d" % (sb, n_sub, L), data, DECODE, coef)
            e["sub_bits"] = sb
            out.append(e)
    for cat in range(10, 16):
        data, coef = long_units(cat)
        e = _entry("long_units_%d" % (16 + cat), data, DECODE if cat <= 11 else J.UNSUPPORTED, coef)
        e["sub_bits"] = 32
        out.append(e)
    return out


def families():
    """-> {family: [entry]}; an entry is dict(name, data, expect, coef) (coef: the coefficients the file codes, None when
    token lists replace some blocks)."""
    return dict(dense=dense(), guard=guard_edges(), colour=[colour_file(v) for v in LUMA_LEVELS], upsampling=upsampling(),
                huffman=huffman_edges(), sync=sync_adversaries())
