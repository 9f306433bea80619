"""GPU: `python -m smap_b200.run_inference` under torchrun's variables (smap_b200.run_inference.run_distributed).

The result file written at any world size must be byte-identical to the one-GPU file for the same flags and images.
The fixture directory holds 11 images (not a multiple of world * batch, so the last step is ragged and at world 2 one
rank has only padding in it): baseline and progressive JPEGs, PNGs, a .jpg the GPU decoders leave to cv2.imread, a flat
grey image (no person to find), and files in sub-directories.

 * world 1 under RANK / WORLD_SIZE / LOCAL_RANK, on every machine: the file equals the plain CLI's with the default
   flags, with --do_flip 1 and -rp, with --glob_order 1, and in fp16 with weights that clamp (the clamp count printed
   must equal the plain CLI's, which checks that the zero frames padding the last step are not counted);
 * world 2, and 8 where the machine has 8 GPUs: the same comparisons;
 * one rank reading a file that neither decoder nor cv2 reads: every rank exits with 1, none reports the file as
   written, and no process of any rank is left."""
import os
import re
import signal
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import preprocess_case_image, refine_state_dict  # noqa: E402

from smap_b200 import schema  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH = 2
CONFIGS = {
    "plain": [],
    "flip_refine": ["--do_flip", "1", "-rp", "{refine}"],
    "glob_order": ["--glob_order", "1"],
    "fp16_clamping": ["--precision", "fp16", "-p", "{smap_hot}"],
}


@pytest.fixture(scope="module")
def fixture(tmp_path_factory):
    cv2 = pytest.importorskip("cv2")
    root = tmp_path_factory.mktemp("dist_cli")
    data = root / "imgs"
    (data / "sub" / "deep").mkdir(parents=True)
    prog = [int(cv2.IMWRITE_JPEG_QUALITY), 90, int(cv2.IMWRITE_JPEG_PROGRESSIVE), 1]
    files = {
        "base0.jpg": (1, []), "b/base1.jpg": (3, []), "sub/base2.jpeg": (5, []), "sub/deep/base3.jpg": (6, []),
        "prog0.jpg": (0, prog), "sub/prog1.jpg": (4, prog),
        "p0.png": (7, []), "sub/p1.png": (2, []), "sub/deep/p2.png": (8, []),
    }
    for name, (ci, params) in files.items():
        (data / name).parent.mkdir(parents=True, exist_ok=True)
        assert cv2.imwrite(str(data / name), preprocess_case_image(ci), params)
    # PNG bytes behind a .jpg name: both GPU decoders refuse it, cv2.imread reads it by its signature
    ok, png = cv2.imencode(".png", preprocess_case_image(9))
    assert ok
    (data / "sub" / "cv2_only.jpg").write_bytes(png.tobytes())
    assert cv2.imwrite(str(data / "flat.png"), np.full((480, 640, 3), 128, np.uint8))
    (data / "notes.txt").write_text("not an image")
    sd = schema.make_state_dict(0, "identity")
    torch.save({"model": sd}, root / "smap.pth")
    hot = dict(sd)
    first = schema.unit_specs(3)[0][0] + ".conv.weight"
    hot[first] = sd[first] * 1e5  # activations far beyond +-65504 from the first layer on: fp16 clamps
    torch.save({"model": hot}, root / "smap_hot.pth")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in refine_state_dict().items()}, root / "refine.pth")
    return root


def _args(root, config, out_dir):
    a = ["-p", str(root / "smap.pth"), "--dataset_path", str(root / "imgs"), "--batch_size", str(BATCH),
         "--json_name", config, "--output_dir", str(out_dir)]
    a += [x.format(refine=root / "refine.pth", smap_hot=root / "smap_hot.pth") for x in CONFIGS[config]]
    return a


def _result(out_dir, config):
    return open(os.path.join(out_dir, "stage3_root2_run_inference_test_%s.json" % config), "rb").read()


def _clamped(text):
    m = re.search(r"fp16: (\d+) activation values exceeded", text)
    return int(m.group(1)) if m else 0


@pytest.fixture(scope="module")
def plain(fixture):
    """The one-GPU CLI without torchrun's variables: config -> (result file bytes, clamp count printed)."""
    out = {}
    for config in CONFIGS:
        out_dir = fixture / "plain" / config
        p = subprocess.run([sys.executable, "-m", "smap_b200.run_inference"] + _args(fixture, config, out_dir), cwd=ROOT,
                           env=_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert p.returncode == 0, p.stdout[-4000:]
        assert "Pairs writed to" in p.stdout and "(11 images)" in p.stdout, p.stdout[-2000:]
        out[config] = (_result(out_dir, config), _clamped(p.stdout))
    assert out["fp16_clamping"][1] > 0, "the fp16 weights were meant to clamp"
    return out


def _env(**extra):
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE")}
    env["SMAPB_NO_AUTOTUNE"] = "1"  # every handle takes the committed tile table: the bytes must not depend on a timing
    env.update(extra)
    return env


def _alive(pgid):
    try:
        os.killpg(pgid, 0)
        return True
    except ProcessLookupError:
        return False


def run_ranks(world, args, log_dir, timeout=900):
    """One `python -m smap_b200.run_inference` per rank with torchrun's variables, each in a session of its own.
    -> (exit codes, outputs, whether any process of a rank's session outlived its rank).  Killed at the timeout."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.makedirs(log_dir, exist_ok=True)
    procs, logs = [], []
    try:
        for rank in range(world):
            env = _env(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), LOCAL_WORLD_SIZE=str(world),
                       MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            logs.append(open(os.path.join(log_dir, "rank%d.log" % rank), "w+"))
            procs.append(subprocess.Popen([sys.executable, "-m", "smap_b200.run_inference"] + args, cwd=ROOT, env=env,
                                          stdout=logs[-1], stderr=subprocess.STDOUT, start_new_session=True))
        deadline = time.monotonic() + timeout
        while any(p.poll() is None for p in procs) and time.monotonic() < deadline:
            time.sleep(0.2)
        codes = [p.poll() for p in procs]
        time.sleep(1.0)
        leftover = any(_alive(p.pid) for p in procs)
    finally:
        for p in procs:
            if _alive(p.pid):
                os.killpg(p.pid, signal.SIGKILL)
            p.wait()
        texts = []
        for f in logs:
            f.seek(0)
            texts.append(f.read())
            f.close()
    return codes, texts, leftover


def _check_world(world, fixture, plain):
    for config in CONFIGS:
        out_dir = fixture / ("w%d" % world) / config
        codes, texts, leftover = run_ranks(world, _args(fixture, config, out_dir), out_dir / "logs")
        report = "\n".join("--- rank %d (exit %s)\n%s" % (r, c, t[-3000:]) for r, (c, t) in enumerate(zip(codes, texts)))
        assert codes == [0] * world, report
        assert not leftover, "a process outlived its rank\n" + report
        assert "Pairs writed to" in texts[0] and "(11 images)" in texts[0], report
        assert all("Pairs writed" not in t for t in texts[1:]), "only rank 0 writes the file"
        want, clamped = plain[config]
        assert _result(out_dir, config) == want, "world %d, %s: the result file differs from the one-GPU file" % (world, config)
        assert _clamped(texts[0]) == clamped, "world %d, %s: fp16 clamp total %d, one GPU %d" % (
            world, config, _clamped(texts[0]), clamped)
        print("\nworld %d %s: %d bytes identical, fp16 clamps %d" % (world, config, len(want), clamped))


def test_world_1_under_torchrun_variables_writes_the_one_gpu_file(fixture, plain):
    import json

    res = json.loads(plain["plain"][0])
    names = [p["image_path"] for p in res["3d_pairs"]]
    print("\nplain CLI: %d of 11 images with persons (%s), %d persons" % (
        len(names), ", ".join(names), sum(len(p["pred_3d"]) for p in res["3d_pairs"])))
    _check_world(1, fixture, plain)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="world 2 needs >= 2 GPUs")
def test_world_2_writes_the_one_gpu_file(fixture, plain):
    _check_world(2, fixture, plain)


@pytest.mark.skipif(torch.cuda.device_count() < 8, reason="world 8 needs 8 GPUs")
def test_world_8_writes_the_one_gpu_file(fixture, plain):
    _check_world(8, fixture, plain)


def test_an_unreadable_file_stops_every_rank(fixture, tmp_path):
    """zz_broken.png sorts last: frame 11 of 12, which at world 2 and batch 2 is rank 1's second frame of step 2."""
    import shutil

    world = min(2, torch.cuda.device_count())
    data = tmp_path / "imgs"
    shutil.copytree(fixture / "imgs", data)
    (data / "zz_broken.png").write_bytes(b"\x89PNG\r\n\x1a\n" + bytes(100))
    out_dir = tmp_path / "out"
    args = ["-p", str(fixture / "smap.pth"), "--dataset_path", str(data), "--batch_size", str(BATCH), "--output_dir",
            str(out_dir)]
    codes, texts, leftover = run_ranks(world, args, tmp_path / "logs", timeout=300)
    report = "\n".join("--- rank %d (exit %s)\n%s" % (r, c, t[-3000:]) for r, (c, t) in enumerate(zip(codes, texts)))
    assert codes == [1] * world, report
    assert not leftover, "a process outlived its rank\n" + report
    assert all("Pairs writed" not in t for t in texts), report
    assert "cannot read image " + str(data / "zz_broken.png") in texts[world - 1], report
    if world > 1:
        assert "stopped: 1 other rank(s) failed" in texts[0], report
