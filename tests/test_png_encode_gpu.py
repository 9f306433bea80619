"""GPU: Engine.encode_png (smapb_encode_png) against cv2.imencode(".png") on the corpus, with skeleton overlays and 3D
panels (oracle/render_numpy.py, oracle/view3d_numpy.py), and run_inference --vis_dir --vis_format png end to end."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import preprocess_case_image  # noqa: E402
from png_encode_corpus import corpus  # noqa: E402

from oracle import render_numpy  # noqa: E402
from oracle import view3d_numpy as V  # noqa: E402
from smap_b200 import schema  # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def cv_png(img):
    ok, b = cv2.imencode(".png", img)
    assert ok
    return b.tobytes()


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=2, in_h=512, in_w=832)
    yield e
    e.close()


def test_corpus_in_batches_of_one_and_eight_equals_cv2(eng):
    named = corpus()
    frames = [f for _, f in named]
    want = [cv_png(f) for f in frames]
    order = np.random.default_rng(0).permutation(len(frames))  # mixed sizes in every batch of 8
    for lo in range(0, len(frames), 8):
        idx = order[lo:lo + 8]
        dev = [torch.from_numpy(frames[i]).cuda() for i in idx]
        before = [d.clone() for d in dev]
        got = eng.encode_png(dev)
        for i, g in zip(idx, got):
            assert g == want[i], named[i][0]
        for d, b in zip(dev, before):
            assert torch.equal(d, b), "an input frame was modified"
    for i in range(len(frames)):  # host frames, uploaded, one per call
        assert eng.encode_png([frames[i]])[0] == want[i], named[i][0]


def test_output_reads_back_as_the_composite(eng):
    frames = [f for name, f in corpus() if f.size < 3 * 10 ** 6][::5]
    for f, data in zip(frames, eng.encode_png(frames)):
        assert np.array_equal(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR), f)
        assert np.array_equal(eng.decode_png([data])[0].cpu().numpy(), f)


def _records(rng, frames, n_persons, in_h=512, in_w=832):
    from oracle import lift_numpy
    from smap_b200.engine import RECORD_DTYPE, scale_row

    rec = np.zeros(len(frames), RECORD_DTYPE)
    scales = np.zeros((len(frames), 9))
    for i, (f, n) in enumerate(zip(frames, n_persons)):
        H, W = f.shape[:2]
        scales[i] = scale_row(lift_numpy.default_scale(W, H))
        rec[i]["count"] = n
        p2, p3 = rec[i]["pred2d"], rec[i]["pred3d"]
        p2[:n, :, 0] = rng.uniform(-40, in_w + 40, (n, 15))
        p2[:n, :, 1] = rng.uniform(-40, in_h + 40, (n, 15))
        p2[:n, :, 3] = np.where(rng.random((n, 15)) < 0.8, rng.uniform(0.1, 3, (n, 15)), 0)
        p2[:n // 2, :, :2] = rng.normal([in_w / 2, in_h / 2], 30, (n // 2, 15, 2))
        p3[:n, :, :3] = rng.normal([0, -20, 400], [70, 90, 120], (n, 15, 3))
        p3[:n, :, 3] = 1
    return rec, scales


def _dev(rec):
    return torch.from_numpy(rec.view(np.uint8).reshape(len(rec), -1)).cuda()


def test_overlay_and_panel_equal_cv2_of_the_oracle_composite(eng):
    rng = np.random.default_rng(31)
    frames = [preprocess_case_image(i) for i in (1, 5, 8)] + [rng.integers(0, 256, s, np.uint8) for s in
                                                              ((1080, 1920, 3), (333, 97, 3), (9, 13, 3), (2, 3, 3))]
    rec, scales = _records(rng, frames, [127, 3, 0, 127, 40, 2, 1])
    sc = torch.from_numpy(scales).cuda()
    got = eng.encode_png([torch.from_numpy(f).cuda() for f in frames], _dev(rec), sc)
    for i, f in enumerate(frames):
        drawn = render_numpy.render(f, rec[i], scales[i])
        assert got[i] == cv_png(drawn), (i, f.shape)
        if i < 3:
            assert np.array_equal(eng.decode_png([got[i]])[0].cpu().numpy(), drawn)
    assert got[2] == eng.encode_png(frames[2:3])[0], "a record with no person gives the plain encoding"
    got = eng.encode_png(frames, _dev(rec), sc, view3d=True)
    for i, f in enumerate(frames):
        assert got[i] == cv_png(V.render_view3d(f, rec[i], scales[i])), (i, f.shape)


def test_infer_device_records(eng):
    from smap_b200.engine import records_to_numpy

    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    frames = [preprocess_case_image(i) for i in (1, 8)]
    x, sc = eng.preprocess(frames)
    rec = eng.infer_device(x, sc.cuda())
    recs = records_to_numpy(rec)
    print("\ninfer_device persons:", recs["count"].tolist())
    got = eng.encode_png(frames, rec, sc)
    for i, f in enumerate(frames):
        assert got[i] == cv_png(render_numpy.render(f, recs[i], sc[i].numpy()))
    got = eng.encode_png(frames, rec, sc, view3d=True)
    for i, f in enumerate(frames):
        assert got[i] == cv_png(V.render_view3d(f, recs[i], sc[i].numpy()))


def test_bad_arguments_are_refused_and_change_nothing(eng):
    f = np.random.default_rng(4).integers(0, 256, (5, 7, 3), np.uint8)
    good = eng.encode_png([f])[0]
    lib, st = eng.lib, eng._st()

    def call(frames, rec=None, sc=None, flags=0):
        ptrs = (ctypes.c_void_p * len(frames))(*[t.data_ptr() for t in frames])
        hs = (ctypes.c_int * len(frames))(*[t.shape[0] for t in frames])
        ws = (ctypes.c_int * len(frames))(*[t.shape[1] for t in frames])
        sizes = (ctypes.c_int64 * len(frames))()
        rc = lib.smapb_encode_png(eng._h, len(frames), ptrs, hs, ws, rec, sc, flags, sizes, st)
        return rc, lib.smapb_last_error(eng._h).decode()

    wide = torch.zeros(1, 16385, 3, dtype=torch.uint8, device="cuda")
    small = torch.from_numpy(f).cuda()
    rc, msg = call([small, wide])
    assert rc == -1 and "frame 1" in msg and "16384" in msg
    rc, msg = call([small], flags=1)
    assert rc == -1 and "records" in msg
    rc, msg = call([small], flags=2)
    assert rc == -1 and "flags" in msg
    rec, scales = _records(np.random.default_rng(5), [f], [3])
    bad = scales.copy()
    bad[0, 1] += 1
    rc, msg = call([small], ctypes.c_void_p(_dev(rec).data_ptr()), ctypes.c_void_p(torch.from_numpy(bad).cuda().data_ptr()))
    assert rc == -1 and "scale row of frame 0" in msg
    p, n = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_int64()
    assert lib.smapb_encoded_png(eng._h, 0, ctypes.byref(p), ctypes.byref(n)) == 0
    assert ctypes.string_at(p, n.value) == good, "a refused call keeps the previous files"
    assert lib.smapb_encoded_png(eng._h, 1, ctypes.byref(p), None) == -1
    assert eng.encode_png([small])[0] == good == cv_png(f)


def test_launch_count_does_not_depend_on_size_or_content(eng):
    rng = np.random.default_rng(6)
    counts = []
    for frames in ([np.zeros((1, 1, 3), np.uint8)], [rng.integers(0, 256, (1080, 1920, 3), np.uint8)],
                   [np.full((3024, 4032, 3), 7, np.uint8), rng.integers(0, 256, (7, 5, 3), np.uint8), np.zeros((100, 1, 3), np.uint8)]):
        dev = [torch.from_numpy(f).cuda() for f in frames]
        before = eng.launch_count()
        eng.encode_png(dev)
        counts.append(eng.launch_count() - before)
    print("\nlaunches per call:", counts)
    assert len(set(counts)) == 1


@pytest.fixture(scope="module")
def vis_data(tmp_path_factory):
    root = tmp_path_factory.mktemp("vis_png_cli")
    data = root / "imgs"
    (data / "sub").mkdir(parents=True)
    for name, ci in (("base.jpg", 1), ("p.png", 13), ("sub/q.jpeg", 5)):
        assert cv2.imwrite(str(data / name), preprocess_case_image(ci))
    torch.save({"model": schema.make_state_dict(0, "identity")}, root / "smap.pth")
    return root


def _cli_args(root, out, extra=()):
    return ["-p", str(root / "smap.pth"), "--dataset_path", str(root / "imgs"), "--batch_size", "2", "--json_name", "v",
            "--output_dir", str(out)] + list(extra)


def test_cli_vis_format_png_one_gpu(vis_data, monkeypatch):
    from smap_b200.engine import Engine, records_to_numpy
    from smap_b200.run_inference import image_name, list_images, main

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # the CLI's handle and this one must choose the same tile shapes
    root = vis_data
    assert main(_cli_args(root, root / "plain")) == 0
    assert main(_cli_args(root, root / "vis", ["--vis_dir", str(root / "vis_out"), "--vis_format", "png"])) == 0
    json_name = "stage3_root2_run_inference_test_v.json"
    assert (root / "plain" / json_name).read_bytes() == (root / "vis" / json_name).read_bytes()
    paths = list_images(str(root / "imgs"))
    written = sorted(str(p.relative_to(root / "vis_out")) for p in (root / "vis_out").rglob("*") if p.is_file())
    assert written == sorted(os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".png" for p in paths)
    e = Engine(0, max_batch=2, in_h=512, in_w=832)
    try:
        e.load_state_dict(schema.make_state_dict(0, "identity"))
        for lo in range(0, len(paths), 2):
            frames = [cv2.imread(p, cv2.IMREAD_COLOR) for p in paths[lo:lo + 2]]
            x, sc = e.preprocess(frames)
            recs = records_to_numpy(e.infer_device(x, sc.cuda()))
            for k, p in enumerate(paths[lo:lo + 2]):
                name = os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".png"
                drawn = render_numpy.render(frames[k], recs[k], sc[k].numpy())
                assert (root / "vis_out" / name).read_bytes() == cv_png(drawn), name
                assert np.array_equal(cv2.imread(str(root / "vis_out" / name), cv2.IMREAD_COLOR), drawn)
    finally:
        e.close()


def test_cli_vis_format_png_under_torchrun_writes_the_one_gpu_files(vis_data):
    from test_run_inference_dist_gpu import run_ranks

    root = vis_data
    if not (root / "vis_out").exists():
        pytest.skip("needs test_cli_vis_format_png_one_gpu's files")
    out = root / "w1"
    codes, texts, leftover = run_ranks(1, _cli_args(root, out, ["--vis_dir", str(out / "vis"), "--vis_format", "png",
                                                                 "--batch_size", "1"]), out / "logs")
    assert codes == [0] and not leftover, "\n".join(t[-3000:] for t in texts)
    json_name = "stage3_root2_run_inference_test_v.json"
    assert (out / json_name).read_bytes() == (root / "plain" / json_name).read_bytes()
    want = {str(p.relative_to(root / "vis_out")): p.read_bytes() for p in (root / "vis_out").rglob("*") if p.is_file()}
    got = {str(p.relative_to(out / "vis")): p.read_bytes() for p in (out / "vis").rglob("*") if p.is_file()}
    assert got == want
