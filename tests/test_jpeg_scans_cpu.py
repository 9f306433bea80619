"""CPU: the lossless transcoder round-trips under cv2 on every scan script; the multi-scan oracle (oracle/jpeg_scans_numpy.py)
equals cv2.imread byte for byte on a seeded progressive and multi-scan sequential corpus; smapb_jpeg_info_ex
(SMAPB_JPEG_SCANS) gives cv2's shape and the oracle's status; libjpeg-turbo's block smoothing, bogus progressions, late
DQTs and files over 64 scans are refused; the multi-scan header walk survives damaged headers."""
import numpy as np
import pytest

from jpeg_corpus import SAMPLINGS, content, cv2_jpeg
from jpeg_scans import (SCRIPT_LIBJPEG, SCRIPTS, SEQUENTIAL, corpus, cv2_progressive, damaged, eob_32767, eob_flood,
                        for_components, scan_cap, sos_offsets, transcode, transcoded)
from oracle import jpeg_scans_numpy as S

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def info(b):
    from smap_b200.engine import jpeg_info

    return jpeg_info(b, scans=True)


def scan_params(b, sos):
    ns = b[sos + 4]
    t = sos + 5 + 2 * ns
    return b[t], b[t + 1], b[t + 2] >> 4, b[t + 2] & 15  # Ss, Se, Ah, Al


def scan_end(b, sos):
    """Offset of the marker that ends the scan starting at `sos`."""
    q = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    while True:
        q = b.find(b"\xff", q)
        if b[q + 1] == 0 or 0xD0 <= b[q + 1] <= 0xD7:
            q += 2
            continue
        return q


def drop_scan(b, pred):
    """The file without the first scan whose (Ss, Se, Ah, Al) satisfies pred."""
    for s in sos_offsets(b):
        if pred(*scan_params(b, s)):
            return b[:s] + b[scan_end(b, s):]
    raise AssertionError("no such scan")


@pytest.fixture(scope="module")
def files():
    return corpus() + transcoded() + [("eob_32767", eob_32767()), ("eob_flood", eob_flood()), ("scans_64", scan_cap(64))]


def test_transcoder_round_trips_under_cv2():
    """Needs no decoder of ours: every complete script, sequential or progressive, with and without restart intervals,
    decodes under cv2 to the original file's pixels."""
    rng = np.random.default_rng(22)
    for samp in list(SAMPLINGS) + ["gray"]:
        img = content("smooth", 45, 70, rng)
        b = cv2_jpeg(img[:, :, 0].copy(), 85) if samp == "gray" else cv2_jpeg(img, 85, samp)
        ref = cv2_read(b)
        for name, script in SCRIPTS.items():
            for dri in (0, 2):
                t = transcode(b, for_components(script, 1 if samp == "gray" else 3), name not in SEQUENTIAL, dri)
                assert np.array_equal(cv2_read(t), ref), (samp, name, dri)
                assert t.count(b"\xff\xda") == len(for_components(script, 1 if samp == "gray" else 3)), (samp, name)


def test_oracle_equals_cv2_imread(files):
    assert len(files) > 100
    for name, b in files:
        got = S.decode(b)
        ref = cv2_read(b)
        assert got.shape == ref.shape and np.array_equal(got, ref), name


def test_jpeg_info_ex_gives_cv2_shape_and_the_oracle_status(files):
    from smap_b200.engine import jpeg_info

    for name, b in files:
        st, h, w, o = info(b)
        assert st == 0, name
        assert (h, w) == cv2_read(b).shape[:2], name
        assert (st, h, w, o) == S.info(b), name
        if b"\xff\xc2" in b[:sos_offsets(b)[0]]:
            assert jpeg_info(b)[0] != 0, name  # the plain walk still refuses progressive files


def test_unrefined_low_coefficients_are_refused_because_cv2_smooths_them(monkeypatch):
    """Cut a progressive file after its first scans: coefficients 1..9 are left unrefined, libjpeg-turbo smooths the
    blocks, and cv2's output differs from the plain IDCT of the same coefficients; both walks refuse it.  Dropping only
    the DC refinement scan leaves DC at Al > 0 and every AC coefficient refined: no smoothing, decoded, equal to cv2."""
    b = cv2_progressive(content("smooth", 64, 96, np.random.default_rng(3)), 90, "420")
    sos = sos_offsets(b)
    for k in range(1, len(sos)):
        cut = b[:sos[k]] + b"\xff\xd9"
        assert info(cut)[0] != 0 and S.info(cut)[0] != 0, k
    cut = b[:sos[len(sos) // 2]] + b"\xff\xd9"
    ref = cv2_read(cut)
    with monkeypatch.context() as mp:
        mp.setattr(S, "SAVED_COEFS", 1)
        plain = S.decode(cut)
    assert ref is not None and not np.array_equal(plain, ref)
    nodcref = drop_scan(b, lambda ss, se, ah, al: ss == 0 and ah > 0)
    assert info(nodcref)[0] == 0 and S.info(nodcref)[0] == 0
    assert np.array_equal(S.decode(nodcref), cv2_read(nodcref))


def test_smoothing_rule_on_transcoded_scripts(monkeypatch):
    """The same rule on scripts the transcoder writes.  Luma AC 1..63 left at Al = 1: refused, and cv2's smoothed output
    differs from the plain IDCT.  Only luma 10..63 left at Al = 1, or only DC at Al = 1: no smoothing, decoded, equal to
    cv2."""
    b = cv2_jpeg(content("smooth", 64, 96, np.random.default_rng(6)), 90, "420")
    unrefined = transcode(b, SCRIPT_LIBJPEG[:-1])
    assert info(unrefined)[0] != 0 and S.info(unrefined)[0] != 0
    with monkeypatch.context() as mp:
        mp.setattr(S, "SAVED_COEFS", 1)
        assert not np.array_equal(S.decode(unrefined), cv2_read(unrefined))
    high_only = [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 9, 0, 1), ((0,), 10, 63, 0, 1), ((1,), 1, 63, 0, 0),
                 ((2,), 1, 63, 0, 0), ((0,), 1, 9, 1, 0)]
    dc_only = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 63, 0, 0), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)]
    for script in (high_only, dc_only):
        t = transcode(b, script)
        assert info(t)[0] == 0 and S.info(t)[0] == 0
        assert np.array_equal(S.decode(t), cv2_read(t))
        assert not np.array_equal(cv2_read(t), cv2_read(b))  # information really is missing


def test_scan_cap():
    ok, over = scan_cap(64), scan_cap(65)
    assert info(ok)[0] == 0 and S.info(ok)[0] == 0 and np.array_equal(S.decode(ok), cv2_read(ok))
    assert info(over)[0] != 0 and S.info(over)[0] != 0 and cv2_read(over) is not None


def test_sequential_multi_scan_rules():
    """A component in two sequential scans, or in none, is refused."""
    b = cv2_jpeg(content("noise", 16, 24, np.random.default_rng(9)), 90, "420")
    for script in ([((0,), 0, 63, 0, 0), ((1,), 0, 63, 0, 0)], [((0,), 0, 63, 0, 0), ((0, 1, 2), 0, 63, 0, 0)]):
        t = transcode(b, script, progressive=False)
        assert info(t)[0] != 0 and S.info(t)[0] != 0


def test_bogus_progressions_and_late_dqt_are_refused():
    b = cv2_progressive(content("noise", 37, 61, np.random.default_rng(4)), 90, "444")
    # an AC first scan dropped: the refinement that follows it expects Ah = 0 (libjpeg warns: bogus progression)
    bogus = drop_scan(b, lambda ss, se, ah, al: ss > 0 and ah == 0)
    assert info(bogus)[0] != 0 and S.info(bogus)[0] != 0
    assert cv2_read(bogus) is not None
    # Al > 13, Ah != Al + 1, Se < Ss: rewritten in the first AC scan's header
    s = [o for o in sos_offsets(b) if scan_params(b, o)[0] > 0][0]
    t = s + 5 + 2 * b[s + 4]
    for patch in ((t + 2, 0x0E), (t + 2, 0x31), (t, 10), (t + 1, 64)):
        c = bytearray(b)
        c[t + 2] = b[t + 2]
        c[patch[0]] = patch[1]
        assert info(bytes(c))[0] != 0 and S.info(bytes(c))[0] != 0, patch
    # a DQT that redefines a table the first scan latched
    q = b.find(b"\xff\xdb")
    dqt = b[q:q + 2 + ((b[q + 2] << 8) | b[q + 3])]
    s2 = sos_offsets(b)[1]
    late = b[:s2] + dqt + b[s2:]
    assert info(late)[0] != 0 and S.info(late)[0] != 0
    assert cv2_read(late) is not None


def test_damaged_files_are_refused_or_equal_cv2():
    n_ok = 0
    for name, b in damaged():
        st = info(b)[0]
        assert st == S.info(b)[0] or (st != 0 and S.info(b)[0] != 0), name
        if st != 0:
            continue
        try:
            got = S.decode(b)
        except S.NotDecoded:
            continue
        ref = cv2_read(b)
        assert ref is not None and np.array_equal(got, ref), name
        n_ok += 1
    assert n_ok < len(damaged())


def test_multi_scan_header_fuzz_never_accepts_a_broken_header():
    """Truncation at every byte of the first headers and around every later scan header, byte flips in every scan
    header, overlong segment lengths: the walk never crashes and accepts a file only when the oracle's walk does."""
    rng = np.random.default_rng(12)
    b = cv2_progressive(content("noise", 9, 17, rng), 90, "420", rst=2)
    sos = sos_offsets(b)
    for cut in list(range(0, sos[0] + 12)) + [s + d for s in sos[1:] for d in range(-4, 12)]:
        assert info(b[:cut])[0] != 0, cut
    heads = set(range(2, sos[0] + 12))
    for s in sos[1:]:
        heads |= set(range(s, s + 14))
    for pos in sorted(heads):
        for x in (0x01, 0x80, 0xFF):
            c = bytearray(b)
            c[pos] ^= x
            c = bytes(c)
            assert (info(c)[0] == 0) == (S.info(c)[0] == 0), (pos, x)
    for s in sos:
        c = bytearray(b)
        c[s + 2:s + 4] = b"\xff\xf0"
        assert info(bytes(c))[0] != 0
