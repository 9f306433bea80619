"""Frames/s of the whole run_inference CLI, from image files on disk to the result file, at world 1, 2 and 8 (tools only).

A seeded directory of q90 4:2:0 1920x1080 JPEGs (16 distinct photo-like frames written --frames times under distinct
names in sub-directories) and a checkpoint of seeded weights are made in a temporary directory.  Each world size that
the machine has GPUs for runs `python -m torch.distributed.run --standalone --nproc_per_node W -m smap_b200.run_inference`
twice: over all frames and over a short directory of 2 * W * batch frames.  The CLI's steady rate is the difference in
frames over the difference in wall time, which takes out process start, torch import, weight upload, communicator
set-up and graph capture; the end-to-end wall time of the long run is reported too.  The plain CLI (no torchrun) is
timed the same way as the one-GPU baseline.  The GPUs' name, power limit and SM clock are read in the same call.

    python tools/run_inference_scaling.py [--frames 1024] [--batch 8] [--precision bf16x3] [--worlds 1,2,8]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from jpeg_corpus import content, cv2_jpeg  # noqa: E402
from smap_b200 import schema  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return [l.strip() for l in q.stdout.strip().split("\n") if l.strip()]


def make_dir(path, n, frames):
    for i in range(n):
        d = os.path.join(path, "seq%02d" % (i // 64))
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "f%05d.jpg" % i), "wb") as f:
            f.write(frames[i % len(frames)])


def time_cli(world, data, ckpt, out_dir, args):
    cli = ["-m", "smap_b200.run_inference", "-p", ckpt, "--dataset_path", data, "--output_dir", out_dir] + args
    if world == 0:  # the plain CLI
        cmd = [sys.executable] + cli
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc_per_node", str(world)] + cli
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    t0 = time.perf_counter()
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3600)
    dt = time.perf_counter() - t0
    if p.returncode != 0 or "Pairs writed to" not in p.stdout:
        raise SystemExit("world %d failed (exit %d):\n%s" % (world, p.returncode, p.stdout[-4000:]))
    return dt


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=8, help="--batch_size of the CLI: frames per GPU and step")
    ap.add_argument("--precision", default="bf16x3")
    ap.add_argument("--worlds", default="1,2,8")
    ap.add_argument("--json", default="", help="also write the results here")
    a = ap.parse_args()
    ngpu = torch.cuda.device_count()
    if ngpu < 1:
        raise SystemExit("no CUDA device: this tool measures the CLI on the GPU")
    worlds = [w for w in map(int, a.worlds.split(",")) if w <= ngpu]
    rng = np.random.default_rng(5)
    frames = [cv2_jpeg(content("smooth", 1080, 1920, rng), 90, "420") for _ in range(16)]
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = os.path.join(tmp, "smap.pth")
        torch.save({"model": schema.make_state_dict(0, "identity")}, ckpt)
        big = os.path.join(tmp, "big")
        make_dir(big, a.frames, frames)
        args = ["--batch_size", str(a.batch), "--precision", a.precision]
        for world in [0] + worlds:
            g = max(1, world)
            n0 = 2 * g * a.batch
            short = os.path.join(tmp, "short%d" % world)
            make_dir(short, n0, frames)
            t_short = time_cli(world, short, ckpt, os.path.join(tmp, "out_s%d" % world), args)
            t_long = time_cli(world, big, ckpt, os.path.join(tmp, "out_l%d" % world), args)
            r = dict(world=world if world else 1, launcher="plain" if world == 0 else "torchrun", frames=a.frames,
                     batch_per_gpu=a.batch, precision=a.precision, wall_s=round(t_long, 2), short_wall_s=round(t_short, 2),
                     steady_fps=round((a.frames - n0) / max(1e-9, t_long - t_short), 1),
                     end_to_end_fps=round(a.frames / t_long, 1))
            print(json.dumps(r), flush=True)
            results.append(r)
    info = gpu_info()
    print(json.dumps(dict(gpus=info)))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(gpus=info, results=results), f, indent=1)


if __name__ == "__main__":
    main()
