"""CPU: the PNG decoder's oracle (oracle/png_numpy.py) equals cv2.imdecode byte for byte on a seeded corpus and refuses every
file cv2 refuses; the library's host-only chunk walk (smapb_png_info) agrees with the oracle's; the block oracle
(oracle/inflate_numpy.py) inflates like zlib and its finder rule lists every dynamic block start."""
import struct
import zlib

import numpy as np
import pytest

from oracle import inflate_numpy as Z
from oracle import png_numpy as P
from png_corpus import chunk, corpus, damaged, samples, write_png

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    if not b:
        return None  # cv2.imdecode asserts on an empty buffer; cv2.imread of an empty file returns None
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    return corpus()


def test_oracle_equals_cv2_on_the_corpus(files):
    assert len(files) > 180
    for name, b in files:
        st, got = P.decode(b)
        ref = cv2_read(b)
        assert st == P.OK, (name, st)
        assert ref is not None and got.shape == ref.shape and np.array_equal(got, ref), name


def test_oracle_refuses_what_cv2_refuses_and_equals_it_elsewhere():
    refused = 0
    for name, b in damaged():
        st, got = P.decode(b)
        ref = cv2_read(b)
        if ref is None:
            assert st != P.OK, name
        if st == P.OK:
            assert ref is not None and np.array_equal(got, ref), name
        else:
            refused += 1
    assert refused > 40


def test_cv2_rules_the_decoder_copies():
    """The pixel rules png.cu implements, each pinned on a hand-built file: 16-bit high bytes, dropped alpha, ignored tRNS,
    gAMA and sBIT, 2-bit grey scaling, black for palette indices past PLTE, eXIf rotation, and the refusals."""
    def png(w, h, depth, ctype, rows, pre=b"", z=None):
        raw = b"".join(b"\x00" + r for r in rows)
        return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, 0)) + pre +
                chunk(b"IDAT", zlib.compress(raw) if z is None else z) + chunk(b"IEND", b""))

    v = np.array([256, 0x80ff, 0xfe80], ">u2").tobytes()
    assert cv2_read(png(3, 1, 16, 0, [v]))[0, :, 0].tolist() == [1, 128, 254]
    assert cv2_read(png(1, 1, 8, 6, [bytes([1, 2, 3, 0])])).tolist() == [[[3, 2, 1]]]
    assert cv2_read(png(1, 1, 8, 4, [bytes([9, 0])])).tolist() == [[[9, 9, 9]]]
    assert cv2_read(png(4, 1, 2, 0, [bytes([0b00011011])]))[0, :, 0].tolist() == [0, 85, 170, 255]
    pal = png(3, 1, 8, 3, [bytes([0, 1, 5])], pre=chunk(b"PLTE", bytes([9, 8, 7, 6, 5, 4])) + chunk(b"tRNS", b"\x00"))
    assert cv2_read(pal).tolist() == [[[7, 8, 9], [4, 5, 6], [0, 0, 0]]]
    rgb = [bytes(range(9))]
    base = cv2_read(png(3, 1, 8, 2, rgb))
    for extra in (chunk(b"gAMA", struct.pack(">I", 100000)), chunk(b"sBIT", bytes([5, 5, 5])), chunk(b"tRNS", bytes(6))):
        assert np.array_equal(cv2_read(png(3, 1, 8, 2, rgb, pre=extra)), base)
    from png_corpus import exif_chunk

    assert cv2_read(png(3, 2, 8, 2, rgb * 2, pre=exif_chunk(6))).shape == (3, 2, 3)
    for name, b in [(n, b) for n, b in damaged() if n in ("crc_IDAT", "bad_adler", "too_little", "zhdr_cinfo8",
                                                         "unknown_critical")]:
        assert cv2_read(b) is None, name
    for b in (pal, png(3, 2, 8, 2, rgb * 2, pre=exif_chunk(6))):
        st, got = P.decode(b)
        assert st == P.OK and np.array_equal(got, cv2_read(b))


def info(b):
    from smap_b200.engine import png_info

    return png_info(b)


def test_png_info_agrees_with_the_oracle(files):
    for name, b in files + damaged():
        st, H = P.parse(b)
        got = info(b)
        assert got[0] == st, (name, got, st)
        if st == P.OK:
            assert got[1:3] == H["out_shape"] and got[3] == H["orientation"], name
        else:
            assert got[1:] == (0, 0, 0), name


def test_png_info_survives_every_truncation_and_byte_flip():
    s = samples(3, 4, 9, 13, np.random.default_rng(5))
    b = write_png(s, 3, 4, 1)
    for k in range(len(b)):
        for x in (b[:k], b[:k] + bytes([b[k] ^ 0xff]) + b[k + 1:]):
            assert info(x)[0] == P.parse(x)[0], k


def stream(b):
    return P.parse(b)[1]["z"]


def test_block_oracle_inflates_like_zlib_and_the_finder_lists_every_dynamic_block(files):
    types = set()
    n_dyn = 0
    for name, b in files:
        z = stream(b)
        data, blocks = Z.blocks(z)
        assert data == zlib.decompress(z), name
        assert blocks[-1].final and all(not k.final for k in blocks[:-1]), name
        for k in blocks:
            types.add(k.type)
            if k.type == 2:
                assert Z.finder_accepts(z, k.start), (name, k)
                n_dyn += 1
        assert blocks[0].start == 16 and all(a.end == c.start for a, c in zip(blocks, blocks[1:])), name
    assert types == {0, 1, 2} and n_dyn > 100
