"""CPU: the JPEG encoder oracle (oracle/jpeg_encode_numpy.py) byte for byte against cv2.imencode."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from jpeg_encode_corpus import SIZES, corpus, eos_stuffing_frame, frame  # noqa: E402

from oracle import jpeg_encode_numpy as E  # noqa: E402

cv2 = pytest.importorskip("cv2")


def cv_encode(img, q):
    ok, b = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), q])
    assert ok
    return b.tobytes()


@pytest.mark.parametrize("q", [1, 10, 25, 50, 75, 90, 95, 100])
def test_oracle_equals_cv2_on_the_corpus(q):
    for f in corpus():
        assert E.encode(f, q) == cv_encode(f, q), (f.shape, q)


def test_every_quality_on_a_small_frame():
    """Also settles the quantiser: libjpeg-turbo's reciprocal multiplication gives the rounded quotients at every quality."""
    f = frame("noise", 37, 53, 7)
    g = frame("photo", 37, 53, 8)
    for q in range(1, 101):
        assert E.encode(f, q) == cv_encode(f, q), q
        assert E.encode(g, q) == cv_encode(g, q), q


def test_a_12_megapixel_frame():
    f = frame("photo", 3024, 4032, 3)
    assert E.encode(f, 95) == cv_encode(f, 95)


def test_dummy_blocks_of_a_5x5_frame():
    """One real luma block, then three dummy blocks: zero AC and the DC of the block before them."""
    f = frame("noise", 5, 5, 1)
    coef = E.forward_blocks(E.colour_planes(f), 95, 5, 5)
    assert coef.shape == (6, 64)
    assert (coef[1:4, 1:] == 0).all() and (coef[1:4, 0] == coef[0, 0]).all()


def test_end_of_stream_stuffing():
    img, q = eos_stuffing_frame()
    h, w = img.shape[:2]
    _, bits = E.pack(*E.tokens(E.forward_blocks(E.colour_planes(img), q, h, w)))
    data = E.encode(img, q)
    assert bits % 8 and data.endswith(b"\xff\x00\xff\xd9"), "the padded last byte is 0xFF and is stuffed"
    assert data == cv_encode(img, q)


def test_header_length_does_not_depend_on_quality_or_size():
    assert len({len(E.header(q, h, w)) for q in (1, 50, 100) for h, w in SIZES}) == 1


def test_worst_case_bits_per_block_bound():
    """q100 noise stays under BLOCK_BITS_MAX per block, the bound the GPU sizes its entropy buffer with."""
    f = np.random.default_rng(2).integers(0, 256, (64, 64, 3), np.uint8)
    coef = E.forward_blocks(E.colour_planes(f), 100, 64, 64)
    _, lens = E.tokens(coef)
    assert lens.sum() <= len(coef) * E.BLOCK_BITS_MAX


def test_encoder_kernels_do_not_spill():
    """nvcc -Xptxas -v on jpeg_enc.cu: its 12 kernels use no local memory for spills."""
    import shutil
    import subprocess
    import tempfile

    from smap_b200 import build

    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run(["nvcc"] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "jpeg_enc.cu"),
                            "-o", os.path.join(tmp, "e.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    spills = [line for line in p.stdout.splitlines() if "spill" in line]
    assert len(spills) == 12 and all(" 0 bytes spill stores, 0 bytes spill loads" in s for s in spills), p.stdout
