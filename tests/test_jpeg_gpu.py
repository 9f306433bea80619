"""GPU: Engine.decode_jpeg (smapb_decode_jpeg) equals cv2.imread byte for byte, as one mixed-size batch and one image at a
time; damaged files decode to cv2's bytes or are left to cv2; run_inference decodes .jpg files on the GPU and writes the
result file cv2 decoding writes."""
import os

import numpy as np
import pytest
import torch

from jpeg_corpus import corpus, damaged, large_frames, not_decoded, resize_edge_files

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=1)
    yield e
    e.close()


def where(got, ref):
    d = np.argwhere((got != ref).any(-1))
    return "%d pixels differ, first at %s" % (len(d), d[:3].tolist())


def test_decode_equals_cv2_batched_and_one_at_a_time(eng):
    files = corpus(large=True) + large_frames()
    names = [n for n, _ in files]
    data = [b for _, b in files]
    refs = [cv2_read(b) for b in data]
    batched = eng.decode_jpeg(data)
    for name, got, ref in zip(names, batched, refs):
        assert got is not None, name
        got = got.cpu().numpy()
        assert got.shape == ref.shape, name
        assert np.array_equal(got, ref), (name, where(got, ref))
    for name, b, ref in zip(names, data, refs):
        (got,) = eng.decode_jpeg([b])
        assert got is not None, name
        got = got.cpu().numpy()
        assert np.array_equal(got, ref), (name, "single", where(got, ref))


def test_one_launch_per_phase_for_the_batch(eng):
    files = [b for _, b in corpus()[:40]]
    n0 = eng.launch_count()
    eng.decode_jpeg(files)
    n1 = eng.launch_count()
    eng.decode_jpeg(files[:1])
    n2 = eng.launch_count()
    # unstuffing, the sync passes, prefix, write, DC scan, IDCT, colour: the batch of 40 may need more sync passes than
    # one image, never more launches per image
    assert n1 - n0 < 40 and n2 - n1 >= 7


def test_unsupported_and_damaged_files_are_left_to_cv2_or_equal_it(eng):
    bad = not_decoded()
    assert all(o is None for o in eng.decode_jpeg([b for _, b in bad]))
    files = damaged()
    got = eng.decode_jpeg([b for _, b in files])
    n_dec = 0
    for (name, b), g in zip(files, got):
        if g is None:
            continue
        ref = cv2_read(b)
        assert ref is not None and np.array_equal(g.cpu().numpy(), ref), name
        n_dec += 1
    assert n_dec < len(files)
    torch.cuda.synchronize()


def test_run_inference_decodes_jpegs_on_the_gpu(tmp_path, monkeypatch):
    from jpeg_corpus import content, cv2_jpeg, pil_jpeg

    from smap_b200 import schema
    from smap_b200.engine import Engine
    from smap_b200.run_inference import run

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # two handles must choose the same tile shapes for a byte comparison
    rng = np.random.default_rng(4)
    data = tmp_path / "imgs"
    (data / "sub").mkdir(parents=True)
    files = {
        "a.jpg": cv2_jpeg(content("smooth", 360, 640, rng), 90, "420"),
        "sub/b.jpeg": cv2_jpeg(content("noise", 300, 200, rng), 80, "444", rst=4),
        "sub/c.jpg": pil_jpeg(content("smooth", 200, 300, rng), 90, 2, 6),
        "d.jpg": open_progressive(content("smooth", 240, 320, rng)),
    }
    for k, b in files.items():
        (data / k).write_bytes(b)
    assert cv2.imwrite(str(data / "e.png"), content("smooth", 100, 150, rng))
    decoded = []
    real = Engine.decode_jpeg

    def counting(self, blobs):
        out = real(self, blobs)
        decoded.extend(o is not None for o in out)
        return out

    monkeypatch.setattr(Engine, "decode_jpeg", counting)
    sd = schema.make_state_dict(0, "identity")
    got = tmp_path / "gpu.json"
    ref = tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=3) == 5
    assert sum(decoded) == 3 and len(decoded) == 4  # the progressive file went to cv2

    def imread(p):
        return cv2.imread(p, cv2.IMREAD_COLOR)

    assert run(sd, str(data), str(ref), batch_size=3, imread=imread) == 5
    assert len(decoded) == 4  # a caller's imread is used for every file
    assert open(got, "rb").read() == open(ref, "rb").read()
    assert os.path.getsize(got) > 0


def test_decoded_frames_at_the_resizer_edges_preprocess_like_cv2(eng):
    """decode_jpeg -> preprocess on the GPU equals cv2.imdecode -> cv2.resize + letterbox + normalise (cases.cv2_preprocess)
    on 1x1, 7x5 and 17x9 files (up-scaling from 1-pixel sides), a 1663x1024 file and an EXIF-6 file displayed 1664x1023
    (exact 1/2 scale with the last column or row cut)."""
    from cases import cv2_preprocess

    from smap_b200.engine import scale_row

    files = resize_edge_files()
    shapes = set()
    for (name, b), g in zip(files, eng.decode_jpeg([b for _, b in files])):
        ref = cv2_read(b)
        assert g is not None and np.array_equal(g.cpu().numpy(), ref), name
        shapes.add(ref.shape[:2])
        out, scales = eng.preprocess([g])
        want, sc = cv2_preprocess(ref)
        got = out[0].cpu().numpy()
        assert np.array_equal(got, want), (name, "%d values differ" % (got != want).sum())
        assert np.array_equal(scales[0].numpy(), scale_row(sc)), name
    assert {(1, 1), (5, 7), (9, 17), (1024, 1663), (1023, 1664)} <= shapes


def test_run_inference_takes_frames_at_the_resizer_edges(tmp_path, monkeypatch):
    """A directory of 1x1, 7x5, 17x9, 1663x1024 and EXIF-6 1664x1023 JPEGs: every file is decoded on the GPU and
    processed, and the result file equals the one cv2 decoding writes."""
    from smap_b200 import schema
    from smap_b200.run_inference import run

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # two handles must choose the same tile shapes for a byte comparison
    keep = ("1x1_noise_q90_420", "7x5_check_q90_444", "17x9_noise_q50_gray", "1663x1024_noise_q90_420", "exif6_1664x1023_q90_420")
    data = tmp_path / "imgs"
    data.mkdir()
    for name, b in resize_edge_files():
        if name in keep:
            (data / (name + ".jpg")).write_bytes(b)
    assert len(list(data.iterdir())) == len(keep)
    sd = schema.make_state_dict(0, "identity")
    got, ref = tmp_path / "gpu.json", tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=3) == len(keep)
    assert run(sd, str(data), str(ref), batch_size=3, imread=lambda p: cv2.imread(p, cv2.IMREAD_COLOR)) == len(keep)
    assert open(got, "rb").read() == open(ref, "rb").read()


def open_progressive(img):
    import io

    from PIL import Image

    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img[:, :, ::-1])).save(bio, "JPEG", quality=90, progressive=True)
    return bio.getvalue()
