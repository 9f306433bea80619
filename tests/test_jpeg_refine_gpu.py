"""GPU: the split AC refinement (acr_mask_kernel, acr_decode_kernel, acr_apply_kernel in smap_b200/csrc/jpeg.cu) through
Engine.decode_jpeg_ex equals cv2.imread byte for byte, one file at a time and in a shuffled batch with baseline files:
EOB runs of 1..100 blocks at every offset from the decoder's 32-block windows and of 32767 blocks, runs that end at a
restart or at a segment's last block, restart intervals of 1, 3, 32, 33, 65 and none, bands Ss = Se and 1..63, q100 noise
and flat frames, grey and every sampling, 1920x1080 and 4032x3024 frames.  Damaged refinement scans come back None exactly
when the oracle refuses them.  run_inference sends baseline JPEGs to decode_jpeg, progressive ones to decode_jpeg_ex and
the rest to imread, and writes the JSON the cv2 route writes."""
import os

import numpy as np
import pytest
import torch

from jpeg_corpus import content, cv2_jpeg
from jpeg_corpus import corpus as baseline_corpus
from jpeg_scans import cv2_progressive, damaged, large_frames, pil_progressive, transcoded
from oracle import jpeg_scans_numpy as S
from test_jpeg_refine_cpu import refine_damaged, refine_files

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def where(got, ref):
    d = np.argwhere((got != ref).any(-1))
    return "%d pixels differ, first at %s" % (len(d), d[:3].tolist())


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=1)
    yield e
    e.close()


@pytest.fixture(scope="module")
def files():
    return refine_files(large=True) + large_frames() + transcoded()


def test_equals_cv2_one_at_a_time(eng, files):
    for name, b in files:
        (g,) = eng.decode_jpeg_ex([b])
        assert g is not None, name
        g, ref = g.cpu().numpy(), cv2_read(b)
        assert g.shape == ref.shape and np.array_equal(g, ref), (name, where(g, ref))


def test_equals_cv2_in_a_mixed_batch_with_baseline_files(eng, files):
    mixed = files + baseline_corpus()[::5]
    order = np.random.default_rng(3).permutation(len(mixed))
    mixed = [mixed[i] for i in order]
    got = eng.decode_jpeg_ex([b for _, b in mixed])
    for (name, b), g in zip(mixed, got):
        assert g is not None, name
        g, ref = g.cpu().numpy(), cv2_read(b)
        assert g.shape == ref.shape and np.array_equal(g, ref), (name, where(g, ref))


def test_damaged_refinement_scans_are_refused_exactly_when_the_oracle_refuses(eng):
    fs = refine_damaged() + damaged()
    got = eng.decode_jpeg_ex([b for _, b in fs])
    n_none = 0
    for (name, b), g in zip(fs, got):
        try:
            want = S.decode(b)
        except S.NotDecoded:
            want = None
        assert (g is None) == (want is None), name
        if g is None:
            n_none += 1
            continue
        assert np.array_equal(g.cpu().numpy(), want), name
        (one,) = eng.decode_jpeg_ex([b])
        assert one is not None and np.array_equal(one.cpu().numpy(), want), (name, "single")
    assert 100 < n_none < len(fs), (n_none, len(fs))
    torch.cuda.synchronize()


def test_run_inference_routes_progressive_jpegs_to_decode_jpeg_ex(tmp_path, monkeypatch):
    from PIL import Image

    from smap_b200 import schema
    from smap_b200.engine import Engine
    from smap_b200.run_inference import run

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # two handles must choose the same tile shapes for a byte comparison
    rng = np.random.default_rng(8)
    data = tmp_path / "imgs"
    (data / "sub").mkdir(parents=True)
    prog = cv2_progressive(content("smooth", 240, 320, rng), 90, "420")
    sos = [i for i in range(len(prog) - 1) if prog[i] == 0xFF and prog[i + 1] == 0xDA]
    cmyk = __import__("io").BytesIO()
    Image.fromarray(content("smooth", 64, 96, rng)).convert("CMYK").save(cmyk, "JPEG", quality=90)
    files = {
        "a.jpg": cv2_jpeg(content("smooth", 360, 640, rng), 90, "420"),               # baseline: decode_jpeg
        "b.jpg": prog,                                                                 # progressive: decode_jpeg_ex
        "sub/c.jpeg": pil_progressive(content("smooth", 200, 300, rng), 90, 0),       # progressive: decode_jpeg_ex
        "sub/d.jpg": cv2_progressive(content("noise", 90, 130, rng), 90, "444", rst=3),  # progressive: decode_jpeg_ex
        "e.jpg": prog[:sos[len(sos) // 2]] + b"\xff\xd9",  # refinement left out, libjpeg-turbo smooths it: imread
        "f.jpg": cmyk.getvalue(),                                                      # CMYK: imread
    }
    for k, b in files.items():
        (data / k).write_bytes(b)
    assert cv2.imwrite(str(data / "g.png"), content("smooth", 100, 150, rng))
    calls = {"decode_jpeg": [], "decode_jpeg_ex": []}
    for meth in calls:
        real = getattr(Engine, meth)

        def counting(self, blobs, _real=real, _log=calls[meth]):
            out = _real(self, blobs)
            _log.append([o is not None for o in out])
            return out

        monkeypatch.setattr(Engine, meth, counting)
    read = []

    def imread(p):
        read.append(os.path.relpath(p, data))
        return cv2.imread(p, cv2.IMREAD_COLOR)

    import smap_b200.run_inference as ri

    real_read_frames = ri.read_frames
    monkeypatch.setattr(ri, "read_frames", lambda eng, paths, _imread: real_read_frames(eng, paths, imread))
    sd = schema.make_state_dict(0, "identity")
    got, ref = tmp_path / "gpu.json", tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=8) == 7
    assert calls["decode_jpeg"] == [[True] + [False] * 5]  # a, b, e, f, sub/c, sub/d in sorted order
    assert calls["decode_jpeg_ex"] == [[True, True, True]]  # b, sub/c, sub/d
    assert sorted(read) == ["e.jpg", "f.jpg"]  # the PNG went to the GPU PNG decoder
    monkeypatch.setattr(ri, "read_frames", real_read_frames)

    def cv2_imread(p):
        return cv2.imread(p, cv2.IMREAD_COLOR)

    n_ex = len(calls["decode_jpeg_ex"])
    assert run(sd, str(data), str(ref), batch_size=8, imread=cv2_imread) == 7
    assert len(calls["decode_jpeg_ex"]) == n_ex  # a caller's imread is used for every file
    assert open(got, "rb").read() == open(ref, "rb").read()
    assert os.path.getsize(got) > 0


def test_run_inference_records_of_a_progressive_folder_equal_the_cv2_route(tmp_path, monkeypatch):
    """bf16x3 records (the JSON) of 1920x1080 progressive frames, GPU decoding against cv2.imread."""
    from smap_b200 import schema
    from smap_b200.run_inference import run

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")
    rng = np.random.default_rng(9)
    data = tmp_path / "prog"
    data.mkdir()
    for k in range(3):
        (data / ("%d.jpg" % k)).write_bytes(cv2_progressive(content("smooth", 1080, 1920, rng), 90, "420"))
    sd = schema.make_state_dict(0, "identity")
    got, ref = tmp_path / "gpu.json", tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=2, precision="bf16x3") == 3
    assert run(sd, str(data), str(ref), batch_size=2, precision="bf16x3",
               imread=lambda p: cv2.imread(p, cv2.IMREAD_COLOR)) == 3
    assert open(got, "rb").read() == open(ref, "rb").read()
