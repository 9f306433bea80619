"""GPU: Engine.decode_jpeg_ex (smapb_decode_jpeg_ex with SMAPB_JPEG_SCANS) equals cv2.imread byte for byte on progressive
files, in mixed batches with baseline and refused files and one at a time, at the default and at the shortest
subsequence length, including every transcoder script (sequential multi-scan too), an EOB run of 32767, 64 scans and EOB
runs that add up past 2^31 blocks; damaged files decode to cv2's bytes or are refused; the launch count grows with the number of scans,
not with the batch."""
import numpy as np
import pytest
import torch

from jpeg_corpus import content, not_decoded
from jpeg_corpus import corpus as baseline_corpus
from jpeg_scans import (corpus, cv2_progressive, damaged, eob_32767, eob_flood, large_frames, scan_cap, sos_offsets,
                        transcoded)

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def where(got, ref):
    d = np.argwhere((got != ref).any(-1))
    return "%d pixels differ, first at %s" % (len(d), d[:3].tolist())


@pytest.fixture(scope="module")
def files():
    crafted = [("eob_32767", eob_32767()), ("eob_flood", eob_flood()), ("scans_64", scan_cap(64))]
    return corpus(large=True) + large_frames() + transcoded() + crafted


def engine():
    from smap_b200.engine import Engine

    return Engine(0, max_batch=1)


@pytest.mark.parametrize("sub_bits", [None, "32"])
def test_decode_ex_equals_cv2_in_mixed_batches_and_one_at_a_time(files, sub_bits, monkeypatch):
    if sub_bits:
        monkeypatch.setenv("SMAPB_JPEG_SUB_BITS", sub_bits)  # every block crosses subsequence boundaries
    eng = engine()
    try:
        base = baseline_corpus()[::7]
        bad = not_decoded()
        mixed = [(n, b, True) for n, b in files] + [(n, b, True) for n, b in base]
        mixed += [(n, b, False) for n, b in bad if n not in ("progressive", "progressive_cv2")]
        mixed.append(("scans_65", scan_cap(65), False))
        rng = np.random.default_rng(1)
        order = rng.permutation(len(mixed))
        mixed = [mixed[i] for i in order]
        got = eng.decode_jpeg_ex([b for _, b, _ in mixed])
        for (name, b, ok), g in zip(mixed, got):
            if not ok:
                assert g is None, name
                continue
            assert g is not None, name
            g = g.cpu().numpy()
            ref = cv2_read(b)
            assert g.shape == ref.shape and np.array_equal(g, ref), (name, where(g, ref))
        for name, b in files:
            (g,) = eng.decode_jpeg_ex([b])
            assert g is not None, name
            assert np.array_equal(g.cpu().numpy(), cv2_read(b)), (name, "single")
    finally:
        eng.close()


def test_plain_decode_still_refuses_them(files):
    eng = engine()
    try:
        multi = [b for _, b in files if len(sos_offsets(b)) > 1]
        assert all(o is None for o in eng.decode_jpeg(multi))
    finally:
        eng.close()


def test_damaged_files_are_refused_or_equal_cv2():
    """Files whose headers pass and whose entropy-coded data does not decode (runs past Se, refinement symbols of size
    != 1, segments that end short) come back None from the device checks."""
    from smap_b200.engine import jpeg_info

    eng = engine()
    try:
        fs = damaged()
        got = eng.decode_jpeg_ex([b for _, b in fs])
        n_dec = n_device_refused = 0
        for (name, b), g in zip(fs, got):
            if g is None:
                n_device_refused += jpeg_info(b, scans=True)[0] == 0
                continue
            ref = cv2_read(b)
            assert ref is not None and np.array_equal(g.cpu().numpy(), ref), name
            n_dec += 1
        assert n_dec < len(fs) and n_device_refused >= 3
        torch.cuda.synchronize()
    finally:
        eng.close()


def test_launches_depend_on_the_rounds_not_on_the_batch():
    rng = np.random.default_rng(2)
    fs = [cv2_progressive(content("noise", 48, 64, rng), 90, "420") for _ in range(40)]
    rounds = len(sos_offsets(fs[0]))
    eng = engine()
    try:
        n0 = eng.launch_count()
        eng.decode_jpeg_ex(fs[:1])
        n1 = eng.launch_count()
        eng.decode_jpeg_ex(fs)
        n2 = eng.launch_count()
        one, batch = n1 - n0, n2 - n1
        assert one >= rounds + 3
        assert batch <= one + 8 * rounds  # at most one more group of sync passes per round
    finally:
        eng.close()
