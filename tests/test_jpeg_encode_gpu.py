"""GPU: Engine.encode_jpeg (smapb_encode_jpeg) against cv2.imencode and against the overlay oracle
(oracle/jpeg_encode_numpy.py, oracle/render_numpy.py), and run_inference --vis_dir end to end."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import preprocess_case_image  # noqa: E402
from jpeg_encode_corpus import corpus, eos_stuffing_frame  # noqa: E402

from oracle import jpeg_encode_numpy as E  # noqa: E402
from oracle import render_numpy  # noqa: E402
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


def test_batches_of_one_and_eight_equal_cv2(eng):
    frames = corpus()
    for q in (1, 25, 50, 75, 90, 95, 100):
        for lo in range(0, len(frames), 8):
            batch = frames[lo:lo + 8]
            dev = [torch.from_numpy(f).cuda() for f in batch]
            before = [d.clone() for d in dev]
            got = eng.encode_jpeg(dev, q)
            for f, g, d, b in zip(batch, got, dev, before):
                assert g == cv_encode(f, q), (f.shape, q)
                assert torch.equal(d, b), "the input frame was modified"
        one = eng.encode_jpeg([frames[3]], q)  # a host frame, uploaded
        assert one[0] == cv_encode(frames[3], q)


def test_worst_case_and_end_of_stream_stuffing(eng):
    noise = np.random.default_rng(5).integers(0, 256, (1080, 1920, 3), np.uint8)
    got = eng.encode_jpeg([noise], 100)[0]
    assert got == cv_encode(noise, 100)
    nblk = 6 * ((1920 + 15) // 16) * ((1080 + 15) // 16)
    print("\nq100 noise: %d bytes, %.0f%% of the entropy bound" % (len(got), 100 * len(got) / (2 * nblk * E.BLOCK_BITS_MAX / 8)))
    img, q = eos_stuffing_frame()
    got = eng.encode_jpeg([img], q)[0]
    assert got.endswith(b"\xff\x00\xff\xd9") and got == cv_encode(img, q)


def test_output_decodes_like_cv2(eng):
    frames = corpus()[:6]
    for f, data in zip(frames, eng.encode_jpeg(frames, 90)):
        dec = eng.decode_jpeg([data])[0]
        assert np.array_equal(dec.cpu().numpy(), cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR))


def test_bad_arguments_are_refused(eng):
    f = torch.zeros(4, 4, 3, dtype=torch.uint8, device="cuda")
    for q in (0, 101):
        with pytest.raises(Exception, match="quality"):
            eng.encode_jpeg([f], q)
    with pytest.raises(Exception, match="16384"):
        eng.encode_jpeg([torch.zeros(1, 16385, 3, dtype=torch.uint8, device="cuda")], 95)


def _records(rng, frames, n_persons, in_h=512, in_w=832):
    from smap_b200.engine import RECORD_DTYPE, scale_row
    from oracle import lift_numpy

    rec = np.zeros(len(frames), RECORD_DTYPE)
    scales = np.zeros((len(frames), 9))
    for i, (f, n) in enumerate(zip(frames, n_persons)):
        H, W = f.shape[:2]
        scales[i] = scale_row(lift_numpy.default_scale(W, H))
        rec[i]["count"] = n
        p = rec[i]["pred2d"]
        p[:n, :, 0] = rng.uniform(-40, in_w + 40, (n, 15))
        p[:n, :, 1] = rng.uniform(-40, in_h + 40, (n, 15))
        p[:n, :, 3] = np.where(rng.random((n, 15)) < 0.8, rng.uniform(0.1, 3, (n, 15)), 0)
        # persons that overlap: half of them around one spot
        p[:n // 2, :, :2] = rng.normal([in_w / 2, in_h / 2], 30, (n // 2, 15, 2))
    return rec, scales


def _check_overlay(eng, frames, rec, scales, q=95):
    rec_t = torch.from_numpy(rec.view(np.uint8).reshape(len(frames), -1)).cuda()
    got = eng.encode_jpeg([torch.from_numpy(f).cuda() for f in frames], q, rec_t, torch.from_numpy(scales).cuda())
    for i, f in enumerate(frames):
        drawn = render_numpy.render(f, rec[i], scales[i])
        assert got[i] == E.encode(drawn, q), (i, f.shape)
    return got


def test_overlay_equals_the_oracle_on_seeded_records(eng):
    rng = np.random.default_rng(11)
    frames = [preprocess_case_image(i) for i in (1, 5, 8, 13)] + [rng.integers(0, 256, (1080, 1920, 3), np.uint8),
                                                                  rng.integers(0, 256, (333, 97, 3), np.uint8)]
    rec, scales = _records(rng, frames, [127, 3, 0, 40, 127, 5])
    got = _check_overlay(eng, frames, rec, scales)
    plain = eng.encode_jpeg(frames[2:3], 95)[0]
    assert got[2] == plain, "a record with no person gives the plain encoding"
    # a scale row that does not describe the frame is refused
    bad = scales.copy()
    bad[0, 1] += 1
    with pytest.raises(Exception, match="scale row"):
        eng.encode_jpeg(frames[:1], 95, torch.from_numpy(rec[:1].view(np.uint8).reshape(1, -1)).cuda(),
                        torch.from_numpy(bad[:1]).cuda())


def test_overlay_equals_the_oracle_on_infer_device_records(eng):
    from smap_b200.engine import records_to_numpy

    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    frames = [preprocess_case_image(i) for i in (1, 8)]
    x, sc = eng.preprocess(frames)
    rec = eng.infer_device(x, sc.cuda())
    recs = records_to_numpy(rec)
    print("\ninfer_device persons:", recs["count"].tolist())
    got = eng.encode_jpeg(frames, 95, rec, sc)
    for i, f in enumerate(frames):
        assert got[i] == E.encode(render_numpy.render(f, recs[i], sc[i].numpy()), 95)


@pytest.fixture(scope="module")
def vis_data(tmp_path_factory):
    root = tmp_path_factory.mktemp("vis_cli")
    data = root / "imgs"
    (data / "sub").mkdir(parents=True)
    prog = [int(cv2.IMWRITE_JPEG_QUALITY), 90, int(cv2.IMWRITE_JPEG_PROGRESSIVE), 1]
    for name, ci, params in (("base.jpg", 1, []), ("sub/prog.jpg", 8, prog), ("p.png", 13, []), ("sub/q.jpeg", 5, [])):
        assert cv2.imwrite(str(data / name), preprocess_case_image(ci), params)
    ok, png = cv2.imencode(".png", preprocess_case_image(9))  # PNG bytes behind a .jpg name: only cv2.imread reads it
    (data / "sub" / "cv2_only.jpg").write_bytes(png.tobytes())
    torch.save({"model": schema.make_state_dict(0, "identity")}, root / "smap.pth")
    return root


def _cli_args(root, out, extra=()):
    return ["-p", str(root / "smap.pth"), "--dataset_path", str(root / "imgs"), "--batch_size", "2", "--json_name", "v",
            "--output_dir", str(out)] + list(extra)


def test_cli_vis_dir_one_gpu(vis_data, monkeypatch):
    from smap_b200.engine import Engine, records_to_numpy
    from smap_b200.run_inference import image_name, list_images, main

    monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # the CLI's handle and this one must choose the same tile shapes
    root = vis_data
    assert main(_cli_args(root, root / "plain")) == 0
    assert main(_cli_args(root, root / "vis", ["--vis_dir", str(root / "vis_out")])) == 0
    json_name = "stage3_root2_run_inference_test_v.json"
    assert (root / "plain" / json_name).read_bytes() == (root / "vis" / json_name).read_bytes()
    paths = list_images(str(root / "imgs"))
    eng = Engine(0, max_batch=2, in_h=512, in_w=832)
    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    written = sorted(str(p.relative_to(root / "vis_out")) for p in (root / "vis_out").rglob("*") if p.is_file())
    assert written == sorted(os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".jpg" for p in paths)
    for lo in range(0, len(paths), 2):
        frames = [cv2.imread(p, cv2.IMREAD_COLOR) for p in paths[lo:lo + 2]]
        x, sc = eng.preprocess(frames)
        recs = records_to_numpy(eng.infer_device(x, sc.cuda()))
        for k, p in enumerate(paths[lo:lo + 2]):
            name = os.path.splitext(image_name(p, str(root / "imgs")))[0] + ".jpg"
            want = E.encode(render_numpy.render(frames[k], recs[k], sc[k].numpy()), 95)
            assert (root / "vis_out" / name).read_bytes() == want, name
    eng.close()


@pytest.mark.parametrize("world", [1, 2])
def test_cli_vis_dir_under_torchrun_writes_the_one_gpu_files(vis_data, world):
    from test_run_inference_dist_gpu import run_ranks

    if torch.cuda.device_count() < world:
        pytest.skip("world %d needs >= %d GPUs" % (world, world))
    root = vis_data
    if not (root / "vis_out").exists():
        pytest.skip("needs test_cli_vis_dir_one_gpu's files")
    out = root / ("w%d" % world)
    codes, texts, leftover = run_ranks(world, _cli_args(root, out, ["--vis_dir", str(out / "vis"), "--batch_size", "1"]),
                                       out / "logs")
    assert codes == [0] * world and not leftover, "\n".join(t[-3000:] for t in texts)
    want = {str(p.relative_to(root / "vis_out")): p.read_bytes() for p in (root / "vis_out").rglob("*") if p.is_file()}
    got = {str(p.relative_to(out / "vis")): p.read_bytes() for p in (out / "vis").rglob("*") if p.is_file()}
    assert got == want
