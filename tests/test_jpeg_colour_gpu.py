"""GPU: Engine.decode_jpeg_ex(colour=True) (smapb_decode_jpeg_ex with SMAPB_JPEG_SCANS | SMAPB_JPEG_COLOUR) equals
cv2.imread byte for byte on the CMYK / YCCK / RGB / sampling corpus of tests/golden/jpeg_colour.py, refused files come back
None; so it does in one shuffled batch with baseline, progressive and refused files, on 1920x1080 and 4032x3024 frames of
every large kind, and with SMAPB_JPEG_COLOUR alone on the single-scan files.  run(..., jpeg_colour=True) decodes those
files on the GPU and writes the JSON the cv2 route writes."""
import os

import numpy as np
import pytest

from jpeg_colour import DECODE, LARGE_KINDS, corpus, large_frames
from jpeg_corpus import content, cv2_jpeg, not_decoded
from jpeg_corpus import corpus as baseline_corpus
from jpeg_scans import corpus as progressive_corpus
from jpeg_scans import sos_offsets

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def where(got, ref):
    d = np.argwhere((got != ref).any(-1))
    return "%d pixels differ, first at %s" % (len(d), d[:3].tolist())


def check(files, got):
    for (name, b, ok), g in zip(files, got):
        if not ok:
            assert g is None, name
            continue
        assert g is not None, name
        g = g.cpu().numpy()
        ref = cv2_read(b)
        assert g.shape == ref.shape and np.array_equal(g, ref), (name, where(g, ref))


@pytest.fixture(scope="module")
def files():
    return [(n, b, e == DECODE) for n, b, e in corpus()]


def engine():
    from smap_b200.engine import Engine

    return Engine(0, max_batch=1)


def test_corpus_equals_cv2_in_one_batch_and_one_at_a_time(files):
    eng = engine()
    try:
        check(files, eng.decode_jpeg_ex([b for _, b, _ in files], colour=True))
        for f in files[::3]:
            check([f], eng.decode_jpeg_ex([f[1]], colour=True))
        single = [f for f in files if len(sos_offsets(f[1])) == 1 and f[1].find(b"\xff\xc2") < 0]
        check(single, eng.decode_jpeg_ex([b for _, b, _ in single], scans=False, colour=True))
    finally:
        eng.close()


def test_mixed_batch_with_baseline_progressive_refused_and_large_frames(files):
    rng = np.random.default_rng(3)
    mixed = [f for f in files if not f[2]] + [f for f in files if f[2]][::4]
    mixed += [(n, b, True) for n, b in baseline_corpus()[::9]] + [(n, b, True) for n, b in progressive_corpus()[::5]]
    mixed += [(n, b, n in ("cmyk", "411", "rgb", "progressive", "progressive_cv2")) for n, b in not_decoded()]
    for kind in LARGE_KINDS:
        for h, w in ((1080, 1920), (3024, 4032)):
            mixed += [("%s_%dx%d" % (kind, h, w), b, True) for b in large_frames(kind, h, w)]
    mixed = [mixed[i] for i in rng.permutation(len(mixed))]
    eng = engine()
    try:
        check(mixed, eng.decode_jpeg_ex([b for _, b, _ in mixed], colour=True))
    finally:
        eng.close()


def test_without_colour_the_new_frames_stay_refused(files):
    eng = engine()
    try:
        new = [(n, b) for n, b, ok in files if ok and not n.startswith("gray_")]
        assert all(g is None for g in eng.decode_jpeg_ex([b for _, b in new]))
        assert all(g is None for g in eng.decode_jpeg([b for _, b in new]))
    finally:
        eng.close()


def test_run_inference_jpeg_colour_decodes_them_on_the_gpu(tmp_path, monkeypatch):
    from smap_b200 import schema
    from smap_b200.engine import Engine, jpeg_info
    from smap_b200.run_inference import run
    import smap_b200.run_inference as ri

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")
    rng = np.random.default_rng(10)
    data = tmp_path / "imgs"
    data.mkdir()
    named = {n: b for n, b, _ in corpus()}
    files = {
        "a.jpg": cv2_jpeg(content("smooth", 360, 640, rng), 90, "420"),
        "b.jpg": large_frames("cmyk444", 240, 320)[0],
        "c.jpg": large_frames("cmyk420", 200, 300)[0],
        "d.jpeg": large_frames("ycck420", 180, 260)[0],
        "e.jpg": large_frames("ycc411", 230, 310)[0],
        "f.jpg": named["rgb_ids_70x45"],
        "g.jpg": named["pil_rgb_smooth_70x45"],
        "h.jpg": named["ycc_luma_coarse_libjpeg"],
        "i.jpg": named["adobe1_cmyk"],  # left to cv2
    }
    for k, b in files.items():
        (data / k).write_bytes(b)
    calls = []
    real = Engine.decode_jpeg_ex

    def counting(self, blobs, *a, **kw):
        out = real(self, blobs, *a, **kw)
        calls.append(([o is not None for o in out], kw.get("colour")))
        return out

    monkeypatch.setattr(Engine, "decode_jpeg_ex", counting)
    read = []

    def imread(p):
        read.append(os.path.relpath(p, data))
        return cv2.imread(p, cv2.IMREAD_COLOR)

    real_read_frames = ri.read_frames
    monkeypatch.setattr(ri, "read_frames", lambda eng, paths, _imread, **kw: real_read_frames(eng, paths, imread, **kw))
    sd = schema.make_state_dict(0, "identity")
    got, ref = tmp_path / "gpu.json", tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=16, jpeg_colour=True) == len(files)
    assert calls == [([True] * 7, True)]  # b..h; i is refused by the header walk and never sent
    assert read == ["i.jpg"]
    assert jpeg_info(files["i.jpg"], scans=True, colour=True)[0] != 0
    monkeypatch.setattr(ri, "read_frames", real_read_frames)
    assert run(sd, str(data), str(ref), batch_size=16, imread=lambda p: cv2.imread(p, cv2.IMREAD_COLOR)) == len(files)
    assert open(got, "rb").read() == open(ref, "rb").read()
    assert os.path.getsize(got) > 0
