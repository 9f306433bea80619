"""GPU: Engine.decode_jpeg equals cv2.imread byte for byte on the files of tests/golden/jpeg_writer.py (baseline streams
libjpeg never writes), one at a time and in one shuffled batch with the cv2 corpus and the refused files, and through
decode_jpeg_ex; the refused files come back None; and each file decoded alone, the cv2 corpus included, takes the
launches the CPU model of the sync passes predicts, at subsequences of 32, 64 and 512 bits."""
import numpy as np
import pytest

import jpeg_writer as W
from jpeg_corpus import corpus, not_decoded

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")

MODEL_BYTES = 1 << 16  # files whose launches are predicted (the model decodes in Python)


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    fs = [e for f in W.families().values() for e in f]
    for i, (n, b) in enumerate(corpus()):  # cv2's files: their launch counts too (a quarter of them at 32 and 64 bits)
        fs.append(dict(name=n, data=b, expect=W.DECODE, model_all=i % 4 == 0))
    for e in fs:
        e["ref"] = cv2_read(e["data"])
    return fs


def engine(monkeypatch, sub_bits=None):
    from smap_b200.engine import Engine

    if sub_bits:
        monkeypatch.setenv("SMAPB_JPEG_SUB_BITS", str(sub_bits))  # read when the decoder's workspace is created
    return Engine(0, max_batch=1)


def check(name, got, e):
    if e["expect"] != W.DECODE:
        assert got is None, name
        return
    assert got is not None, name
    g = got.cpu().numpy()
    ref = e["ref"]
    assert g.shape == ref.shape, name
    d = np.argwhere((g != ref).any(-1))
    assert len(d) == 0, (name, "%d pixels differ, first at %s" % (len(d), d[:3].tolist()))


@pytest.mark.parametrize("ex", [False, True])
def test_shuffled_batch_with_the_corpus_and_the_refused_files(files, ex, monkeypatch):
    """Tables and quantisers differ per image: nothing may leak between the images of a batch."""
    eng = engine(monkeypatch)
    try:
        mixed = [(e["name"], e["data"], e) for e in files]
        mixed += [(n, b, dict(expect=-1)) for n, b in not_decoded() if not (ex and n.startswith("progressive"))]
        order = np.random.default_rng(3).permutation(len(mixed))
        mixed = [mixed[i] for i in order]
        dec = eng.decode_jpeg_ex if ex else eng.decode_jpeg
        got = dec([b for _, b, _ in mixed])
        for (name, _, e), g in zip(mixed, got):
            check(name, g, e)
    finally:
        eng.close()


@pytest.mark.parametrize("sub_bits", [32, 64, 512])
def test_one_at_a_time_with_the_predicted_launches(files, sub_bits, monkeypatch):
    from smap_b200.engine import jpeg_info

    eng = engine(monkeypatch, sub_bits)
    try:
        worst = 0
        for e in files:
            n0 = eng.launch_count()
            (g,) = eng.decode_jpeg([e["data"]])
            n = eng.launch_count() - n0
            check(e["name"], g, e)
            if jpeg_info(e["data"])[0] == 0:  # decoded, or refused on the device after the whole pipeline ran
                if len(e["data"]) <= MODEL_BYTES and (sub_bits == 512 or e.get("model_all", True)):
                    P = W.predicted_passes(e["data"], sub_bits)
                    assert n == P["launches"], (e["name"], n, P)
                    worst += P["worst"] and e.get("sub_bits") == sub_bits
            else:
                assert n == 0, e["name"]  # refused at the header: nothing is launched
        assert worst >= 7
    finally:
        eng.close()
