"""CPU: the JPEG decoder's oracle (oracle/jpeg_numpy.py) equals cv2.imread byte for byte on a seeded corpus, and the library's
host-only header walk (smapb_jpeg_info) gives cv2's shape, refuses what the GPU decoder does not decode, and survives
malformed headers."""
import numpy as np
import pytest

from jpeg_corpus import corpus, damaged, not_decoded, scan_start
from oracle import jpeg_numpy as J

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    return corpus(large=True)


def test_oracle_equals_cv2_imread(files):
    assert len(files) > 300
    for name, b in files:
        got = J.decode(b)
        ref = cv2_read(b)
        assert got.shape == ref.shape and np.array_equal(got, ref), name


def test_idct_saturates_and_leaves_16_bit_overflow_to_cv2(monkeypatch):
    """q100 checkerboards with their quantisers scaled up (16-bit DQT): blocks that overshoot far beyond 0..255.
    Saturation reproduces cv2 where a 10-bit wrap-around range table does not, and the guard refuses those blocks."""
    from jpeg_corpus import content, cv2_jpeg, dqt16

    b = dqt16(cv2_jpeg(content("check", 64, 64, np.random.default_rng(0)), 100, "444"), 8)
    ref = cv2_read(b)
    with pytest.raises(J.NotDecoded) as e:
        J.decode(b)
    assert e.value.status == J.UNSUPPORTED
    monkeypatch.setattr(J, "GUARD", 1 << 15)  # no 16-bit lane overflows at this scale yet
    assert np.array_equal(J.decode(b), ref)
    monkeypatch.setattr(J, "IDCT_CLAMP", False)
    assert not np.array_equal(J.decode(b), ref)


def info(b):
    from smap_b200.engine import jpeg_info

    return jpeg_info(b)


def test_jpeg_info_gives_cv2_shape(files):
    for name, b in files:
        st, h, w, o = info(b)
        assert st == 0, name
        assert (h, w) == cv2_read(b).shape[:2], name
        assert (st, h, w, o) == J.info(b), name


def test_unsupported_inputs_are_not_decoded():
    for name, b in not_decoded():
        st = info(b)[0]
        assert st != 0, name
        assert J.info(b)[0] != 0, name
        assert cv2_read(b) is not None, name  # cv2 reads them: the caller's fallback


def test_damaged_files_are_not_decoded_or_equal_cv2():
    """Header-level: a damaged header is never decodable; a file the header walk accepts decodes (oracle) to cv2's
    bytes or is refused by the entropy decoder."""
    n_ok = 0
    for name, b in damaged():
        st = info(b)[0]
        assert st == J.info(b)[0] or (st != 0 and J.info(b)[0] != 0), name
        if st != 0:
            continue
        try:
            got = J.decode(b)
        except J.NotDecoded:
            continue
        ref = cv2_read(b)
        assert ref is not None and np.array_equal(got, ref), name
        n_ok += 1
    assert n_ok < len(damaged())


def test_header_fuzz_never_accepts_a_broken_header():
    """Truncation at every byte of the headers, single-byte flips there, overlong segment lengths: the header walk never
    crashes and accepts a file only when the oracle's walk does too."""
    from jpeg_corpus import content, cv2_jpeg, pil_jpeg

    rng = np.random.default_rng(11)
    bases = [cv2_jpeg(content("noise", 9, 17, rng), 90, "420", rst=2), pil_jpeg(content("smooth", 16, 24, rng), 80, 1, 6)]
    for b in bases:
        s0 = scan_start(b)
        for cut in range(0, s0 + 4):
            assert info(b[:cut])[0] != 0, cut
        for pos in range(2, s0):
            for x in (0x01, 0x80, 0xFF):
                c = bytearray(b)
                c[pos] ^= x
                c = bytes(c)
                st = info(c)[0]
                assert (st == 0) == (J.info(c)[0] == 0), (pos, x)
        # every segment length made to overrun the file
        p = 2
        while True:
            m = b[p + 1]
            c = bytearray(b)
            c[p + 2:p + 4] = b"\xff\xf0"
            assert info(bytes(c))[0] != 0, hex(m)
            p += 2 + ((b[p + 2] << 8) | b[p + 3])
            if m == 0xDA:
                break
    assert info(b"")[0] != 0 and info(b"\xff\xd8")[0] != 0 and info(b"\xff\xd8\xff")[0] != 0
