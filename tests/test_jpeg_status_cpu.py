"""CPU: the exact status smapb_jpeg_info_ex gives files with one or two header defects, with flags 0 and with
SMAPB_JPEG_SCANS.  The two modes check some things at different points of the walk (SOF2, the pixel cap, the colour
space, the SOS component count and length, what follows the first scan, Huffman tables that do not build), so a file
with two defects can get a different code in each.  Callers route files by these codes, so they stay as they are."""
import numpy as np
import pytest

from jpeg_corpus import content, cv2_jpeg
from jpeg_scans import cv2_progressive, sos_offsets

pytest.importorskip("cv2")

OK, UNSUPPORTED, MALFORMED, CORRUPT, TOO_LARGE = 0, 1, 2, 3, 4


def segments(b):
    """(offset, marker, length field) of every marker segment up to and including the first SOS."""
    out, p = [], 2
    while True:
        m, L = b[p + 1], (b[p + 2] << 8) | b[p + 3]
        out.append((p, m, L))
        if m == 0xDA:
            return out
        p += 2 + L


def segment(b, marker):
    p, _, L = next(s for s in segments(b) if s[1] == marker)
    return p, b[p:p + 2 + L]


def oversized(b):
    """The frame made 9000 x 9000 (over SMAPB_JPEG_MAX_PIXELS), the data left as it is."""
    p, _ = next((p, m) for p, m, _ in segments(b) if m in (0xC0, 0xC1, 0xC2))
    c = bytearray(b)
    c[p + 5:p + 9] = (9000).to_bytes(2, "big") * 2
    return bytes(c)


def adobe_rgb(b):
    """The JFIF APP0 replaced by an Adobe APP14 with transform 0: the three components are RGB."""
    p, app0 = segment(b, 0xE0)
    app14 = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"
    return b[:p] + app14 + b[p + len(app0):]


def oversubscribed(b):
    """Three 1-bit codes in the first Huffman table (moved from a longer length): the code space overflows."""
    p, _ = segment(b, 0xC4)
    counts = bytearray(b[p + 5:p + 21])
    j = next(j for j in range(1, 16) if counts[j] >= 3)
    counts[j] -= 3
    counts[0] += 3
    return b[:p + 5] + bytes(counts) + b[p + 21:]


def sos_components(b, ns):
    """The first SOS rewritten to name only the first ns components, with a length that matches."""
    p, sos = segment(b, 0xDA)
    head = bytes([ns]) + sos[5:5 + 2 * ns] + sos[-3:]
    return b[:p] + b"\xff\xda" + (2 + len(head)).to_bytes(2, "big") + head + b[p + len(sos):]


def sos_patch(b, offset, value):
    p, _ = segment(b, 0xDA)
    c = bytearray(b)
    c[p + offset] = value
    return bytes(c)


def before_eoi(b, seg):
    assert b.endswith(b"\xff\xd9")
    return b[:-2] + seg + b[-2:]


def rst_out_of_sequence(b):
    """The first restart marker made RST1 instead of RST0."""
    i = b.find(b"\xff\xd0", sos_offsets(b)[0])
    assert i > 0
    return b[:i + 1] + b"\xd1" + b[i + 2:]


def cases():
    rng = np.random.default_rng(31)
    base = cv2_jpeg(content("noise", 24, 40, rng), 90, "420", rst=1)
    prog = cv2_progressive(content("noise", 24, 40, rng), 90, "420")
    _, dht = segment(base, 0xC4)
    p_sos = segment(base, 0xDA)[0]
    sos_and_data = base[p_sos:-2]
    sos_len = (base[p_sos + 2] << 8) | base[p_sos + 3]
    # (name, file, status with flags 0, status with SMAPB_JPEG_SCANS)
    return [
        ("base", base, OK, OK),
        ("progressive", prog, UNSUPPORTED, OK),
        ("sof2_oversized", oversized(prog), UNSUPPORTED, TOO_LARGE),
        ("oversized_adobe_rgb", oversized(adobe_rgb(base)), UNSUPPORTED, TOO_LARGE),
        ("adobe_rgb", adobe_rgb(base), UNSUPPORTED, UNSUPPORTED),
        ("oversized_oversubscribed", oversized(oversubscribed(base)), TOO_LARGE, TOO_LARGE),
        ("sos_one_of_three", sos_components(base, 1), UNSUPPORTED, CORRUPT),
        ("sos_count_one_length_three", sos_patch(base, 4, 1), UNSUPPORTED, MALFORMED),
        ("sos_length_plus_two", sos_patch(base, 3, sos_len + 2), UNSUPPORTED, MALFORMED),
        ("app0_after_scan", before_eoi(base, b"\xff\xe0\x00\x04ab"), UNSUPPORTED, UNSUPPORTED),
        ("app2_after_scan", before_eoi(base, b"\xff\xe2\x00\x04ab"), UNSUPPORTED, OK),
        ("dht_after_scan", before_eoi(base, dht), UNSUPPORTED, OK),
        ("second_sos", before_eoi(base, sos_and_data), UNSUPPORTED, UNSUPPORTED),
        ("oversubscribed", oversubscribed(base), MALFORMED, MALFORMED),
        ("oversubscribed_rst_out_of_sequence", oversubscribed(rst_out_of_sequence(base)), CORRUPT, MALFORMED),
        ("rst_out_of_sequence", rst_out_of_sequence(base), CORRUPT, CORRUPT),
    ]


def test_status_codes_of_each_mode():
    from smap_b200.engine import jpeg_info

    for name, b, st0, st_scans in cases():
        assert jpeg_info(b)[0] == st0, name
        assert jpeg_info(b, scans=True)[0] == st_scans, name
