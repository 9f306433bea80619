"""CPU: SMAPB_JPEG_COLOUR's frames (CMYK, YCCK, RGB, every integral sampling).  The oracle (oracle/jpeg_colour_numpy.py)
equals cv2.imread byte for byte on the seeded corpus of tests/golden/jpeg_colour.py; smapb_jpeg_info_ex with
SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR gives the oracle's status and cv2's shape; without the flag every file keeps the status
the baseline and multi-scan walks give it; fractional ratios, 11 blocks per MCU, 2 components and the Adobe transforms
libjpeg only warns about are refused; run_inference's --jpeg_colour reaches run()."""
import numpy as np
import pytest
import torch

from jpeg_colour import DECODE, REFUSED, corpus
from jpeg_scans import sos_offsets
from oracle import jpeg_colour_numpy as O
from oracle import jpeg_numpy as J
from oracle import jpeg_scans_numpy as S

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    return corpus()


def test_oracle_equals_cv2(files):
    n = 0
    for name, b, expect in files:
        ref = cv2_read(b)
        if expect != DECODE:
            assert O.info(b)[0] == expect, name
            if name in REFUSED:
                assert ref is None, name  # cv2 refuses these too
            continue
        assert ref is not None, name
        got = O.decode(b)
        assert got.shape == ref.shape and np.array_equal(got, ref), name
        n += 1
    assert n >= 250


def test_info_with_colour_gives_the_oracle_status_and_cv2_shape(files):
    from smap_b200.engine import jpeg_info

    for name, b, expect in files:
        st, h, w, o = jpeg_info(b, scans=True, colour=True)
        assert (st, h, w, o) == O.info(b), name
        assert (st == 0) == (expect == DECODE), name
        if st == 0:
            assert (h, w) == cv2_read(b).shape[:2], name


def test_without_colour_every_file_keeps_its_status(files):
    """flags 0 and SMAPB_JPEG_SCANS: the baseline and multi-scan oracles' statuses, which the existing walks give; only
    grayscale frames (whatever their factors) were decoded before."""
    from smap_b200.engine import jpeg_info

    for name, b, _ in files:
        plain, multi = jpeg_info(b)[0], jpeg_info(b, scans=True)[0]
        assert plain == J.info(b)[0], name
        assert multi == S.info(b)[0], name
        assert (plain == 0 or multi == 0) == name.startswith("gray_"), name


def test_colour_alone_widens_the_single_scan_walk(files):
    from smap_b200.engine import jpeg_info

    for name, b, _ in files:
        st = jpeg_info(b, colour=True)[0]
        if len(sos_offsets(b)) == 1 and b[b.find(b"\xff\xc0"):][:2] == b"\xff\xc0":
            assert st == jpeg_info(b, scans=True, colour=True)[0], name
        else:
            assert st == J.UNSUPPORTED, name  # progressive or several scans: SMAPB_JPEG_SCANS is needed


def test_refused_frames(files):
    from smap_b200.engine import jpeg_info

    refused = {name: b for name, b, expect in files if expect != DECODE}
    assert set(REFUSED) | {"adobe1_cmyk", "adobe3_cmyk"} == set(refused)
    for name, b in refused.items():
        assert jpeg_info(b, scans=True, colour=True)[0] == J.UNSUPPORTED, name


def test_unknown_flags_are_rejected():
    from smap_b200 import _lib
    from smap_b200.engine import SmapB200Error, _header_info

    b = corpus()[0][1]
    with pytest.raises(SmapB200Error):
        _header_info(_lib.load().smapb_jpeg_info_ex, b, 4)


@pytest.mark.parametrize("flag", [None, "0", "1"])
def test_cli_passes_jpeg_colour_through(tmp_path, monkeypatch, flag):
    from smap_b200 import run_inference as R

    ckpt = tmp_path / "SMAP.pth"
    torch.save({"model": {}}, str(ckpt))
    got = {}

    def fake_run(*args, **kw):
        got.update(kw)
        return 0

    monkeypatch.setattr(R, "run", fake_run)
    argv = ["-p", str(ckpt), "--dataset_path", str(tmp_path), "--output_dir", str(tmp_path / "out")]
    if flag:
        argv += ["--jpeg_colour", flag]
    assert R.main(argv) == 0
    assert got["jpeg_colour"] is (flag == "1")  # off by default
