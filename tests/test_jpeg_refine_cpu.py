"""CPU: a numpy model of the GPU decoder's split AC refinement (smap_b200/csrc/jpeg.cu: acr_mask_kernel, acr_decode_kernel,
acr_apply_kernel) equals the multi-scan oracle (oracle/jpeg_scans_numpy.py) coefficient for coefficient, and refuses
exactly the files the oracle refuses.  The model keeps the device's word layout: per block of a refinement scan, in the
scan's order, a history mask (bit k = zig-zag coefficient k of [Ss, Se] is nonzero before the scan), the correction bits
(bit i for the i-th history coefficient) and the new +-2^Al coefficients as a position mask and a sign mask.

The files built here (EOB runs of chosen lengths around the decoder's 32-block windows, restart intervals, bands, dense
and empty histories, damaged refinement scans) are the GPU test's too (tests/test_jpeg_refine_gpu.py)."""
import numpy as np
import pytest

from jpeg_corpus import SAMPLINGS, content, cv2_jpeg
from jpeg_scans import corpus, cv2_progressive, damaged, pil_progressive, sos_offsets, transcode, transcoded
from oracle import jpeg_numpy as J
from oracle import jpeg_scans_numpy as S

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")

ZZ = J.ZIGZAG.tolist()
# EOB runs (in blocks) the run files hold, in this order: each length at several offsets from a 32-block window's start
RUNS = [1, 31, 32, 33, 64, 65, 1, 1, 2, 31, 33, 32, 65, 64, 5, 100, 31, 32, 33, 1, 64, 65, 3, 32]
DC_AC_REFINE = [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((0,), 1, 63, 1, 0)]


# ---- the model ---------------------------------------------------------------------------------------------------------
def is_ac_refinement(sc):
    return sc["ah"] > 0 and sc["ss"] > 0


def history_masks(coef, hd, sc):
    """-> uint64 [blocks of the scan]: bit k set when zig-zag coefficient k lies in [Ss, Se] and is nonzero."""
    n = sc["nmcu"] * sc["bpm"]
    blk = coef[[S._block_index(hd, sc, b) for b in range(n)]][:, ZZ]
    ks = np.arange(sc["ss"], sc["se"] + 1)
    return ((blk[:, ks] != 0).astype(np.uint64) << ks.astype(np.uint64)).sum(1, dtype=np.uint64)


def _take_lsb(bits, n):
    """The next n bits as a word whose bit i is the i-th of them."""
    v = 0
    for a in range(0, n, 32):
        k = min(32, n - a)
        v = (v << k) | bits.get(k)
    return int("{:0{}b}".format(v, n)[::-1], 2) if n else 0


def refine_records(data, hd, sc, masks):
    """acr_decode_kernel: -> ([(corr, pos, neg)] per block in scan order, the EOB run lengths read).  Raises
    NotDecoded(CORRUPT) where the device sets SMAPB_JPEG_CORRUPT."""
    d = bytes(data)
    ss, se = sc["ss"], sc["se"]
    lut = J._huff_table(*sc["ac"][0])
    n = sc["nmcu"] * sc["bpm"]
    per = (sc["dri"] or sc["nmcu"]) * sc["bpm"]
    recs, runs = [None] * n, []
    for si, (a, b) in enumerate(sc["segments"]):
        bits = S._Bits(J._unstuff(d[a:b]))
        run = 0
        for blk in range(si * per, min(n, (si + 1) * per)):
            m = int(masks[blk])
            if run:
                recs[blk] = (_take_lsb(bits, bin(m).count("1")), 0, 0)
                run -= 1
                continue
            corr = nc = newp = newn = 0
            k = ss
            while k <= se:
                sym = bits.huff(lut)
                r, s = sym >> 4, sym & 15
                eob = neg = False
                if s:
                    if s != 1:
                        raise S.NotDecoded(S.CORRUPT, "refinement symbol with size != 1")
                    neg = bits.get(1) == 0
                elif r != 15:
                    run = (1 << r) + bits.get(r) - 1
                    runs.append(run + 1)
                    eob, t = True, se + 1
                if not eob:
                    zeros = [z for z in range(k, se + 1) if not (m >> z) & 1]
                    t = zeros[r] if len(zeros) > r else se + 1
                    if s and t > se:
                        raise S.NotDecoded(S.CORRUPT, "run past Se")
                nb = bin(m & ((1 << t) - (1 << k))).count("1")
                corr |= _take_lsb(bits, nb) << nc
                nc += nb
                if s:
                    newp |= 1 << t
                    newn |= neg << t
                if eob:
                    break
                k = t + 1
            recs[blk] = (corr, newp, newn)
    return recs, runs


def apply_records(coef, hd, sc, masks, recs):
    """acr_apply_kernel, in place on int64 coefficients."""
    p1 = 1 << sc["al"]
    for b, (corr, newp, newn) in enumerate(recs):
        blk = coef[S._block_index(hd, sc, b)]
        m, i = int(masks[b]), 0
        for k in range(64):
            if (m >> k) & 1:
                if (corr >> i) & 1 and (int(blk[ZZ[k]]) & p1) == 0:
                    blk[ZZ[k]] += p1 if blk[ZZ[k]] >= 0 else -p1
                i += 1
            if (newp >> k) & 1:
                blk[ZZ[k]] = -p1 if (newn >> k) & 1 else p1


def model_coefficients(data):
    """-> (int16 coefficients after every scan, EOB run lengths of the refinement scans).  Other scans are the oracle's,
    one at a time; refinement scans go through masks -> records -> apply."""
    hd = S.parse(data)
    bpm = sum(c[1] * c[2] for c in hd["comps"])
    coef = np.zeros((hd["nmcu"] * bpm, 64), np.int64)
    runs = []
    for sc in hd["scans"]:
        if is_ac_refinement(sc):
            masks = history_masks(coef, hd, sc)
            recs, r = refine_records(data, hd, sc, masks)
            apply_records(coef, hd, sc, masks, recs)
            runs += r
        else:
            one = S.entropy_decode(data, dict(hd, scans=[sc])).astype(np.int64)
            coef = coef | one if sc["ah"] else coef + one
    return coef.astype(np.int16), runs


def oracle_coefficients(data):
    return S.entropy_decode(data, S.parse(data))


# ---- files -------------------------------------------------------------------------------------------------------------
def runs_file(runs, dri=0, hist=0.5, seed=41):
    """A grayscale file whose AC refinement scan (DC, AC 1..63 at Al = 1, then its refinement) holds EOB runs of the given
    lengths in order, the last one running to the frame's last block.  A run starts at a block with a new +-1 (zig-zag 1..40);
    a share `hist` of the blocks carries a +-2 / +-3 (one correction bit).  dri: restart interval in blocks (libjpeg's
    encoder ends a run at every restart)."""
    rng = np.random.default_rng(seed)
    total = sum(runs)
    nbw = min(total, 128)
    nbh = -(-total // nbw)
    n = nbw * nbh
    coef = np.zeros((n, 64), np.int64)
    coef[:, 0] = rng.integers(-20, 21, n)
    has = np.flatnonzero(rng.random(n) < hist)
    coef[has, J.ZIGZAG[rng.integers(1, 64, len(has))]] = rng.choice([-3, -2, 2, 3], len(has))
    for s0 in np.cumsum([0] + list(runs[:-1])):
        coef[s0, ZZ[int(rng.integers(1, 41))]] = rng.choice([-1, 1])
    from jpeg_writer import write

    return transcode(write(coef, 8 * nbh - 3, 8 * nbw - 5, "gray"), DC_AC_REFINE, dri=dri)


def flat_refine(h=1456, w=1456):
    """A flat grayscale frame of 33124 blocks, every AC coefficient zero: its refinement scan is an EOB run of 32767
    blocks and one of 357, with empty masks."""
    return transcode(cv2_jpeg(np.full((h, w), 77, np.uint8), 90), DC_AC_REFINE)


def band_file(seed=43):
    """Refinement bands Ss = Se (1, 2, 9, 10, 62, 63) and wider ones, on 4:2:0 noise; luma 1..63 refined band by band."""
    b = cv2_jpeg(content("noise", 45, 70, np.random.default_rng(seed)), 95, "420")
    bands = [(1, 1), (2, 2), (3, 8), (9, 9), (10, 10), (11, 61), (62, 62), (63, 63)]
    script = [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((2,), 1, 63, 0, 1)]
    script += [((0,), ss, se, 1, 0) for ss, se in bands] + [((1,), 1, 63, 1, 0), ((2,), 1, 63, 1, 0)]
    return transcode(b, script)


def refine_files(large=False):
    """-> list of (name, bytes) with AC refinement scans, every one decodable (and equal to cv2)."""
    rng = np.random.default_rng(47)
    out = [("runs", runs_file(RUNS)), ("runs_nohist", runs_file(RUNS, hist=0.0, seed=42)),
           ("runs_dense", runs_file(RUNS, hist=1.0, seed=44))]
    for dri in (1, 3, 32, 33, 65):
        out.append(("runs_rst%d" % dri, runs_file(RUNS, dri=dri, seed=45 + dri)))
    out.append(("bands", band_file()))
    for samp in list(SAMPLINGS) + ["gray"]:
        img = content("noise", 61, 83, rng)
        if samp == "gray":
            img = img[:, :, 0].copy()
        for rst in (0, 1, 3):
            out.append(("q100_noise_%s_rst%d" % (samp, rst), cv2_progressive(img, 100, samp, rst=rst)))
        out.append(("q75_noise_%s" % samp, cv2_progressive(img, 75, samp)))
    out.append(("pil_q100_420", pil_progressive(content("noise", 61, 83, rng), 100, 2)))
    if large:
        out.append(("flat_eob_32767", flat_refine()))
        out.append(("flat_1920x1080", cv2_progressive(content("flat", 1080, 1920, rng), 90, "420")))
        out.append(("smooth_1920x1080_420", cv2_progressive(content("smooth", 1080, 1920, rng), 90, "420")))
        out.append(("smooth_1920x1080_rst3", cv2_progressive(content("smooth", 1080, 1920, rng), 90, "422", rst=3)))
        out.append(("noise_4032x3024_420", cv2_progressive(content("noise", 3024, 4032, rng), 90, "420")))
        out.append(("smooth_4032x3024_444", cv2_progressive(content("smooth", 3024, 4032, rng), 90, "444")))
    return out


def refinement_scans(b):
    """-> [(start of the scan's entropy-coded data, its end)] of every AC refinement scan of b."""
    out = []
    for s in sos_offsets(b):
        ns = b[s + 4]
        t = s + 5 + 2 * ns
        if b[t] > 0 and b[t + 2] >> 4:
            q = data = s + 2 + ((b[s + 2] << 8) | b[s + 3])
            while b[q] != 0xFF or b[q + 1] == 0 or 0xD0 <= b[q + 1] <= 0xD7:
                q += 1
            out.append((data, q))
    return out


def refine_damaged(per_scan=10, seed=49):
    """Refinement scans cut short (the later scans kept) and with a flipped byte, at offsets spread over each refinement
    scan's data, in three files (no restart, restart 3, a run file)."""
    rng = np.random.default_rng(seed)
    img = content("noise", 37, 61, rng)
    base = [cv2_progressive(img, 90, "420"), cv2_progressive(img, 95, "444", rst=3), runs_file(RUNS[:8], seed=50)]
    out = []
    for k, b in enumerate(base):
        for j, (a, e) in enumerate(refinement_scans(b)):
            for off in np.unique(np.linspace(a, e - 1, per_scan).astype(int)):
                out.append(("cut%d_scan%d_%d" % (k, j, off), b[:off] + b[e:]))
                c = bytearray(b)
                c[off] ^= int(rng.integers(1, 256))
                out.append(("flip%d_scan%d_%d" % (k, j, off), bytes(c)))
    return out


def outcome(fn, b):
    try:
        return fn(b)
    except S.NotDecoded as e:
        return e.status


# ---- tests -------------------------------------------------------------------------------------------------------------
def test_files_decode_under_cv2_like_the_oracle():
    for name, b in refine_files():
        assert any(is_ac_refinement(sc) for sc in S.parse(b)["scans"]), name
        assert np.array_equal(S.decode(b), cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)), name


def test_run_files_hold_the_runs_they_are_built_for():
    _, runs = model_coefficients(runs_file(RUNS))
    assert runs == RUNS[:-1] + [runs[-1]] and runs[-1] >= RUNS[-1]
    for dri in (32, 33):  # libjpeg's encoder ends every run at a restart: runs that end at a segment's last block
        _, runs = model_coefficients(runs_file(RUNS, dri=dri, seed=45 + dri))
        assert max(runs) == dri and runs.count(dri) >= 3, (dri, runs)
    _, runs = model_coefficients(flat_refine())
    assert runs == [32767, 33124 - 32767]


def test_model_equals_the_oracle():
    files = refine_files() + transcoded() + [(n, b) for n, b in corpus() if n.startswith(("prog_37", "pil_37", "prog_rst"))]
    seen = 0
    for name, b in files:
        hd = S.parse(b)
        seen += any(is_ac_refinement(sc) for sc in hd["scans"])
        got, _ = model_coefficients(b)
        assert np.array_equal(got, oracle_coefficients(b)), name
    assert seen > 50


def test_model_refuses_what_the_oracle_refuses():
    files = damaged() + refine_damaged()
    n_refused = n_ok = 0
    for name, b in files:
        want = outcome(oracle_coefficients, b)
        got = outcome(lambda x: model_coefficients(x)[0], b)
        if isinstance(want, int):
            assert got == want, name
            n_refused += 1
        else:
            assert not isinstance(got, int) and np.array_equal(got, want), name
            n_ok += 1
    assert n_refused > 100 and n_ok > 10, (n_refused, n_ok)
