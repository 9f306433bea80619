"""GPU JPEG encoding (Engine.encode_jpeg) against cv2.imencode, and the run_inference CLI with and without --vis_dir.

    python tools/encode_bench.py [--repeats 3] [--cli_frames 64]

Prints one JSON line per measurement, each with the card's name and power limit read in the same process:
  encode   GPU frames/s for batches of 8 frames (1920x1080 and 4032x3024, q95), plain, with a crowded overlay (127
           persons per frame) and with that overlay plus the 3D panel of the same 127 persons (view3d: an h x (w + h)
           composite per frame), after a warm-up of the same shapes; host clock around calls that end in a device
           synchronisation (encode_jpeg returns once the bytes are on the host);
  cv2      cv2.imencode frames/s on one thread and on every host thread (a thread pool; cv2 releases the GIL);
  cli      run_inference.run frames/s on a directory of 1080p JPEGs (identity weights), bf16x3 and fp16, with and without
           --vis_dir, after one warm-up run of the same configuration.
Each number is repeated --repeats times; min, median and max are reported.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    return q


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 128 + 60 * np.sin(x[..., None] / (37.0 + 13 * np.arange(3))) * np.cos(y[..., None] / 51.0)
    img += rng.normal(0, 4, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def crowd(n, h, w, seed):
    from oracle import lift_numpy
    from smap_b200.engine import RECORD_DTYPE, scale_row

    rng = np.random.default_rng(seed)
    rec = np.zeros(n, RECORD_DTYPE)
    rec["count"] = 127
    rec["pred2d"][..., 0] = rng.uniform(0, 832, (n, 127, 15))
    rec["pred2d"][..., 1] = rng.uniform(0, 512, (n, 127, 15))
    rec["pred2d"][..., 3] = 1
    rec["pred3d"][..., :3] = rng.normal([0, -20, 400], [70, 90, 120], (n, 127, 15, 3))
    rec["pred3d"][..., 3] = 1  # every joint placed, as RefineNet leaves them: 1778 limbs per panel
    sc = np.stack([scale_row(lift_numpy.default_scale(w, h))] * n)
    return torch.from_numpy(rec.view(np.uint8).reshape(n, -1)).cuda(), torch.from_numpy(sc).cuda()


def stats(v):
    v = sorted(v)
    return {"min": round(v[0], 1), "median": round(v[len(v) // 2], 1), "max": round(v[-1], 1)}


def main():
    import cv2

    from smap_b200 import schema
    from smap_b200.engine import Engine
    from smap_b200.run_inference import run

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cli_frames", type=int, default=64)
    ap.add_argument("--skip_cli", action="store_true", help="only the encode and cv2 legs")
    a = ap.parse_args()
    gpu = card()
    eng = Engine(0, max_batch=8)
    B = 8
    for h, w in ((1080, 1920), (3024, 4032)):
        frames = [torch.from_numpy(photo(h, w, s)).cuda() for s in range(B)]
        host = [f.cpu().numpy() for f in frames]
        for overlay, view3d in ((False, False), (True, False), (True, True)):
            extra = crowd(B, h, w, 1) if overlay else (None, None)
            kw = dict(view3d=True) if view3d else {}
            eng.encode_jpeg(frames, 95, *extra, **kw)  # warm-up: workspace growth, module load
            iters = 20 if h == 1080 else 5
            rates = []
            for _ in range(a.repeats):
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(iters):
                    eng.encode_jpeg(frames, 95, *extra, **kw)
                rates.append(iters * B / (time.perf_counter() - t))
            print(json.dumps({"what": "encode", "size": "%dx%d" % (w, h), "batch": B, "overlay": overlay, "view3d": view3d,
                              "frames_per_s": stats(rates), "gpu": gpu}), flush=True)
        for threads in (1, os.cpu_count()):
            cv2.setNumThreads(1)
            rates = []
            for _ in range(a.repeats):
                n = max(threads, 8)
                t = time.perf_counter()
                with ThreadPoolExecutor(threads) as ex:
                    list(ex.map(lambda f: cv2.imencode(".jpg", f, [int(cv2.IMWRITE_JPEG_QUALITY), 95]), host * (n // B + 1)))
                rates.append(B * (n // B + 1) / (time.perf_counter() - t))
            print(json.dumps({"what": "cv2", "size": "%dx%d" % (w, h), "threads": threads, "frames_per_s": stats(rates),
                              "gpu": gpu}), flush=True)
    eng.close()
    if a.skip_cli:
        return
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "imgs")
        os.makedirs(data)
        for i in range(a.cli_frames):
            cv2.imwrite(os.path.join(data, "%04d.jpg" % i), photo(1080, 1920, 100 + i))
        sd = schema.make_state_dict(0, "identity")
        for precision in ("bf16x3", "fp16"):
            for vis in (False, True):
                kw = dict(batch_size=8, precision=precision, vis_dir=os.path.join(tmp, "vis") if vis else None)
                run(sd, data, os.path.join(tmp, "r.json"), **kw)  # warm-up
                rates = []
                for _ in range(a.repeats):
                    t = time.perf_counter()
                    run(sd, data, os.path.join(tmp, "r.json"), **kw)
                    rates.append(a.cli_frames / (time.perf_counter() - t))
                print(json.dumps({"what": "cli", "precision": precision, "vis_dir": vis, "frames": a.cli_frames,
                                  "frames_per_s": stats(rates), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
