"""GPU: Engine.encode_jpeg(view3d=True) (smapb_encode_jpeg_ex with SMAPB_ENCODE_VIEW3D) against cv2.imencode of the
composite oracle (oracle/view3d_numpy.py), and run_inference --vis_dir --vis_3d end to end."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import preprocess_case_image, refine_state_dict  # noqa: E402

from oracle import view3d_numpy as V  # noqa: E402
from smap_b200 import schema  # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def cv_encode(img, q):
    ok, b = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), q])
    assert ok
    return b.tobytes()


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=2, in_h=512, in_w=832)
    yield e
    e.close()


def _records(rng, frames, n_persons, kinds, in_h=512, in_w=832):
    """Seeded records: pred2d as the overlay tests draw them, pred3d of one of these kinds per frame:
    'lift' (joints zeroed with their score, as gen_3d_pose leaves them), 'refine' (every joint placed), 'huge' (spans
    near 1e15, some joints past it), 'flat' (every joint at one point: span 0), 'tiny' (spans of a few ulps and a
    subnormal one, where avail / span overflows)."""
    from oracle import lift_numpy
    from smap_b200.engine import RECORD_DTYPE, scale_row

    rec = np.zeros(len(frames), RECORD_DTYPE)
    scales = np.zeros((len(frames), 9))
    for i, (f, n, kind) in enumerate(zip(frames, n_persons, kinds)):
        H, W = f.shape[:2]
        scales[i] = scale_row(lift_numpy.default_scale(W, H))
        rec[i]["count"] = n
        p2, p3 = rec[i]["pred2d"], rec[i]["pred3d"]
        p2[:n, :, 0] = rng.uniform(-40, in_w + 40, (n, 15))
        p2[:n, :, 1] = rng.uniform(-40, in_h + 40, (n, 15))
        p2[:n, :, 3] = np.where(rng.random((n, 15)) < 0.8, rng.uniform(0.1, 3, (n, 15)), 0)
        p3[:n, :, :3] = rng.normal([0, -20, 400], [70, 90, 120], (n, 15, 3))
        p3[:n // 3, :, :3] = rng.normal([0, -20, 400], 5, (n // 3, 15, 3))  # a third of them in one crowded spot
        p3[:n, :, 3] = p2[:n, :, 3]
        if kind == "lift":
            p3[:n][p2[:n, :, 3] == 0] = 0
        elif kind == "refine":
            p3[:n, :, 3] = 1
        elif kind == "huge":
            p3[:n, :, :3] = rng.uniform(-1e15, 1e15, (n, 15, 3))
            p3[:n, 0, 1] = 3e15
        elif kind == "flat":
            p3[:n, :, :3] = (1.5, -2.25, 300.0)
        elif kind == "tiny":
            p3[:n, :, :3] = 1.0 + rng.integers(0, 4, (n, 15, 3)) * np.finfo(np.float64).eps
            p3[0, :, :3] = rng.integers(0, 2, (15, 3)) * 5e-324
            p3[1:n, :, 3] = 0
    return rec, scales


def _dev(rec):
    return torch.from_numpy(rec.view(np.uint8).reshape(len(rec), -1)).cuda()


def _check(eng, frames, rec, scales, q=95):
    dev = [torch.from_numpy(f).cuda() for f in frames]
    before = [d.clone() for d in dev]
    got = eng.encode_jpeg(dev, q, _dev(rec), torch.from_numpy(scales).cuda(), view3d=True)
    for i, f in enumerate(frames):
        assert got[i] == cv_encode(V.render_view3d(f, rec[i], scales[i]), q), (i, f.shape)
    for d, b in zip(dev, before):
        assert torch.equal(d, b), "an input frame was modified"
    return got


def test_composite_equals_the_oracle_on_seeded_records(eng):
    rng = np.random.default_rng(21)
    frames = [preprocess_case_image(i) for i in (1, 5)] + [rng.integers(0, 256, s, np.uint8) for s in
                                                           ((1080, 1920, 3), (333, 97, 3), (1001, 641, 3), (9, 13, 3),
                                                            (480, 640, 3), (2, 3, 3), (767, 1023, 3))]
    kinds = ["lift", "refine", "refine", "lift", "huge", "flat", "tiny", "refine", "lift"]
    counts = [127, 127, 127, 5, 40, 3, 6, 2, 0]
    rec, scales = _records(rng, frames, counts, kinds)
    _check(eng, frames, rec, scales)
    _check(eng, frames[3:6], rec[3:6], scales[3:6], q=60)


def test_batch_of_eight_equals_eight_batches_of_one(eng):
    rng = np.random.default_rng(22)
    frames = [rng.integers(0, 256, (rng.integers(40, 400), rng.integers(40, 400), 3), np.uint8) for _ in range(8)]
    rec, scales = _records(rng, frames, [127, 0, 3, 60, 1, 127, 9, 20], ["refine", "lift"] * 4)
    batch = _check(eng, frames, rec, scales)
    for i in range(8):
        one = eng.encode_jpeg([frames[i]], 95, _dev(rec[i:i + 1]), torch.from_numpy(scales[i:i + 1]).cuda(), view3d=True)
        assert one[0] == batch[i], i
    plain = eng.encode_jpeg(frames[:2], 95, _dev(rec[:2]), torch.from_numpy(scales[:2]).cuda())
    assert plain[0] != batch[0] and cv2.imdecode(np.frombuffer(plain[0], np.uint8), cv2.IMREAD_COLOR).shape == frames[0].shape


@pytest.mark.parametrize("refine", [False, True])
def test_composite_equals_the_oracle_on_infer_device_records(refine):
    from smap_b200.engine import Engine, records_to_numpy

    e = Engine(0, max_batch=2, in_h=512, in_w=832)
    try:
        e.load_state_dict(schema.make_state_dict(0, "identity"))
        if refine:
            e.load_refine_state_dict(refine_state_dict())
            e.set_refine(True)
        frames = [preprocess_case_image(i) for i in (1, 8)]
        x, sc = e.preprocess(frames)
        rec = e.infer_device(x, sc.cuda())
        recs = records_to_numpy(rec)
        print("\ninfer_device persons:", recs["count"].tolist(), "drawn limbs:", [len(V.drawn_limbs(r)) for r in recs])
        got = e.encode_jpeg(frames, 95, rec, sc, view3d=True)
        for i, f in enumerate(frames):
            assert got[i] == cv_encode(V.render_view3d(f, recs[i], sc[i].numpy()), 95)
    finally:
        e.close()


def test_bad_arguments_are_refused(eng):
    from oracle import lift_numpy
    from smap_b200.engine import RECORD_DTYPE, scale_row

    f = torch.zeros(4, 4, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="records"):
        eng.encode_jpeg([f], 95, view3d=True)
    rec = _dev(np.zeros(1, RECORD_DTYPE))
    for w in (16285, 16284):
        wide = torch.zeros(100, w, 3, dtype=torch.uint8, device="cuda")
        sc = torch.from_numpy(scale_row(lift_numpy.default_scale(w, 100))[None]).cuda()
        if w + 100 > 16384:
            with pytest.raises(Exception, match="frame 0 .*16385"):
                eng.encode_jpeg([wide], 95, rec, sc, view3d=True)
        else:
            got = eng.encode_jpeg([wide], 95, rec, sc, view3d=True)[0]
            assert cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_COLOR).shape == (100, 16384, 3)
    # the C ABI itself: the flag without records, and unknown flag bits
    lib = eng.lib
    ptrs = (ctypes.c_void_p * 1)(f.data_ptr())
    hs, ws, sizes = (ctypes.c_int * 1)(4), (ctypes.c_int * 1)(4), (ctypes.c_int64 * 1)()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.smapb_encode_jpeg_ex(eng._h, 1, ptrs, hs, ws, 95, None, None, 1, sizes, st) == -1
    assert "records" in lib.smapb_last_error(eng._h).decode()
    assert lib.smapb_encode_jpeg_ex(eng._h, 1, ptrs, hs, ws, 95, None, None, 2, sizes, st) == -1
    assert "flags" in lib.smapb_last_error(eng._h).decode()
    assert lib.smapb_encode_jpeg_ex(eng._h, 1, ptrs, hs, ws, 95, None, None, 0, sizes, st) == 0
    assert eng.encode_jpeg([f], 95)[0] == cv_encode(np.zeros((4, 4, 3), np.uint8), 95)


@pytest.fixture(scope="module")
def vis_data(tmp_path_factory):
    root = tmp_path_factory.mktemp("vis3d_cli")
    data = root / "imgs"
    (data / "sub").mkdir(parents=True)
    prog = [int(cv2.IMWRITE_JPEG_QUALITY), 90, int(cv2.IMWRITE_JPEG_PROGRESSIVE), 1]
    portrait = np.ascontiguousarray(preprocess_case_image(5).transpose(1, 0, 2)[:, :-1])
    for name, img, params in (("base.jpg", preprocess_case_image(1), []), ("sub/prog.jpg", preprocess_case_image(8), prog),
                              ("p.png", preprocess_case_image(13), []), ("sub/portrait.jpeg", portrait, [])):
        assert cv2.imwrite(str(data / name), img, params)
    torch.save({"model": schema.make_state_dict(0, "identity")}, root / "smap.pth")
    return root


def _cli_args(root, out, extra=()):
    return ["-p", str(root / "smap.pth"), "--dataset_path", str(root / "imgs"), "--batch_size", "2", "--json_name", "v",
            "--output_dir", str(out)] + list(extra)


JSON_NAME = "stage3_root2_run_inference_test_v.json"


def test_cli_vis_3d_one_gpu(vis_data, monkeypatch):
    from smap_b200.engine import Engine, records_to_numpy
    from smap_b200.run_inference import image_name, list_images, main

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # the CLI's handle and this one must choose the same tile shapes
    root = vis_data
    assert main(_cli_args(root, root / "plain")) == 0
    assert main(_cli_args(root, root / "vis", ["--vis_dir", str(root / "vis_out"), "--vis_3d", "1"])) == 0
    assert (root / "plain" / JSON_NAME).read_bytes() == (root / "vis" / JSON_NAME).read_bytes()
    paths = list_images(str(root / "imgs"))
    written = sorted(str(p.relative_to(root / "vis_out")) for p in (root / "vis_out").rglob("*") if p.is_file())
    assert written == sorted(os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".jpg" for p in paths)
    eng = Engine(0, max_batch=2, in_h=512, in_w=832)
    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    drawn = 0
    for lo in range(0, len(paths), 2):
        frames = [cv2.imread(p, cv2.IMREAD_COLOR) for p in paths[lo:lo + 2]]
        x, sc = eng.preprocess(frames)
        recs = records_to_numpy(eng.infer_device(x, sc.cuda()))
        for k, p in enumerate(paths[lo:lo + 2]):
            name = os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".jpg"
            want = cv_encode(V.render_view3d(frames[k], recs[k], sc[k].numpy()), 95)
            assert (root / "vis_out" / name).read_bytes() == want, name
            drawn += len(V.drawn_limbs(recs[k]))
    eng.close()
    assert drawn > 0, "the fixture's frames draw no 3D limb"


def test_cli_vis_3d_under_torchrun_writes_the_one_gpu_files(vis_data):
    from test_run_inference_dist_gpu import run_ranks

    root = vis_data
    if not (root / "vis_out").exists():
        pytest.skip("needs test_cli_vis_3d_one_gpu's files")
    out = root / "w1"
    codes, texts, leftover = run_ranks(1, _cli_args(root, out, ["--vis_dir", str(out / "vis"), "--vis_3d", "1",
                                                                "--batch_size", "1"]), out / "logs")
    assert codes == [0] and not leftover, "\n".join(t[-3000:] for t in texts)
    want = {str(p.relative_to(root / "vis_out")): p.read_bytes() for p in (root / "vis_out").rglob("*") if p.is_file()}
    got = {str(p.relative_to(out / "vis")): p.read_bytes() for p in (out / "vis").rglob("*") if p.is_file()}
    assert got == want
    assert (out / JSON_NAME).read_bytes() == (root / "plain" / JSON_NAME).read_bytes()
