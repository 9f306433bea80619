"""GPU: Engine.decode_png (smapb_decode_png) equals cv2.imdecode byte for byte in one shuffled mixed batch and one file at a
time; damaged files decode to cv2's bytes or are left to cv2, with the device-side refusals exercised; the inflate
counters show which path ran; run_inference decodes .png files on the GPU and writes the result file cv2 decoding writes."""
import os

import numpy as np
import pytest
import torch

from png_corpus import corpus, damaged, large_frames, samples, write_png

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) if b else None


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=1)
    yield e
    e.close()


def where(got, ref):
    d = np.argwhere((got != ref).any(-1))
    return "%d pixels differ, first at %s" % (len(d), d[:3].tolist())


def test_decode_equals_cv2_in_one_shuffled_mixed_batch_and_one_at_a_time(eng):
    from jpeg_corpus import content, cv2_jpeg

    rng = np.random.default_rng(7)
    good = corpus(large=True) + large_frames(n=2)
    others = [("jpeg", cv2_jpeg(content("smooth", 40, 60, rng))), ("text", b"not an image")] + damaged()
    files = good + others
    order = rng.permutation(len(files))
    batch = [files[i] for i in order]
    got = eng.decode_png([b for _, b in batch])
    n_ok = 0
    for (name, b), g in zip(batch, got):
        ref = cv2_read(b)
        if g is None:
            assert not any(name == n for n, _ in good), name
            continue
        g = g.cpu().numpy()
        assert ref is not None and g.shape == ref.shape and np.array_equal(g, ref), (name, where(g, ref))
        n_ok += 1
    assert n_ok >= len(good)
    for name, b in good:
        (g,) = eng.decode_png([b])
        assert g is not None, name
        assert np.array_equal(g.cpu().numpy(), cv2_read(b)), (name, "single")


def test_damaged_files_are_refused_on_the_device_or_equal_cv2(eng):
    from smap_b200.engine import png_info

    files = damaged()
    got = eng.decode_png([b for _, b in files])
    device_refused = set()
    for (name, b), g in zip(files, got):
        ref = cv2_read(b)
        if g is None:
            if png_info(b)[0] == 0:
                device_refused.add(name)
            continue
        assert ref is not None and np.array_equal(g.cpu().numpy(), ref), name
    # an IDAT CRC, the Adler-32, too little and too much data, a bad filter type: found only once the data is inflated
    assert {"crc_IDAT", "bad_adler", "too_little", "too_much", "bad_filter"} <= device_refused
    torch.cuda.synchronize()


def test_inflate_counters_show_which_path_ran(eng):
    import zlib

    (name, b), = large_frames(n=1, sizes=((1080, 1920),))
    (g,) = eng.decode_png([b])
    st = eng.png_stats()
    assert g is not None and st["confirmed"] > 100 and st["serial"] == 0, st
    assert st["candidates"] >= st["confirmed"] + st["false_positives"] - 1, st
    s = samples(2, 8, 96, 128, np.random.default_rng(3))
    for opts in (dict(level=0), dict(strategy=zlib.Z_FIXED), dict(mem=1), dict(flush=zlib.Z_SYNC_FLUSH, pieces=5)):
        b = write_png(s, 2, 8, zopts=opts)
        (g,) = eng.decode_png([b])
        assert g is not None and np.array_equal(g.cpu().numpy(), cv2_read(b)), opts
        assert eng.png_stats()["serial"] > 0, (opts, eng.png_stats())


def test_launch_count_does_not_grow_with_the_batch(eng):
    files = [b for _, b in corpus()[:60]]
    n0 = eng.launch_count()
    eng.decode_png(files)
    n1 = eng.launch_count()
    eng.decode_png(files[:1])
    n2 = eng.launch_count()
    assert n1 - n0 == n2 - n1 == 8


def test_run_inference_decodes_pngs_on_the_gpu(tmp_path, monkeypatch):
    from jpeg_corpus import content, cv2_jpeg

    from png_corpus import cv2_png, pil_png
    from smap_b200 import schema
    from smap_b200.engine import Engine
    from smap_b200.run_inference import run

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # two handles must choose the same tile shapes for a byte comparison
    rng = np.random.default_rng(9)
    data = tmp_path / "imgs"
    (data / "sub").mkdir(parents=True)
    files = {
        "a.png": cv2_png(content("smooth", 360, 640, rng)),
        "sub/b.png": pil_png(content("noise", 300, 200, rng)),
        "c.png": write_png(samples(3, 4, 240, 320, rng), 3, 4, 1),
        "d.png": write_png(samples(4, 16, 200, 300, rng), 4, 16, 0),
        "e.jpg": cv2_jpeg(content("smooth", 200, 300, rng)),
        "f.png": damaged()[-3][1],  # a PNG cv2 reads but the GPU decoder leaves to it (PLTE in a grey image)
    }
    for k, b in files.items():
        (data / k).write_bytes(b)
    calls = []
    real = Engine.decode_png

    def counting(self, blobs):
        out = real(self, blobs)
        calls.append([o is not None for o in out])
        return out

    monkeypatch.setattr(Engine, "decode_png", counting)
    sd = schema.make_state_dict(0, "identity")
    got, ref = tmp_path / "gpu.json", tmp_path / "cv2.json"
    assert run(sd, str(data), str(got), batch_size=3) == 6
    decoded = sum(calls, [])
    assert len(decoded) == 5 and sum(decoded) == 4
    assert run(sd, str(data), str(ref), batch_size=3, imread=lambda p: cv2.imread(p, cv2.IMREAD_COLOR)) == 6
    assert len(sum(calls, [])) == 5  # a caller's imread is used for every file
    assert open(got, "rb").read() == open(ref, "rb").read()
    assert os.path.getsize(got) > 0
