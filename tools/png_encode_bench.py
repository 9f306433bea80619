"""GPU PNG encoding (Engine.encode_png) against cv2.imencode(".png"), and the run_inference CLI with --vis_format png
against jpg.

    python tools/png_encode_bench.py [--repeats 3] [--cli_frames 32] [--profile]

Prints one JSON line per measurement, each with the card's name and power limit read in the same process:
  encode   GPU frames/s for batches of 8 photo-like frames (1920x1080 and 4032x3024), plain and with a crowded overlay
           (127 persons per frame), after a warm-up of the same shapes; host clock around calls that end in a device
           synchronisation (encode_png returns once the bytes are on the host);
  cv2      cv2.imencode(".png") frames/s on one thread and on 8 host threads (a thread pool; cv2 releases the GIL);
  cli      run_inference.run frames/s on a directory of 1080p JPEGs (identity weights, bf16x3), with --vis_dir in jpg and
           in png, after one warm-up run of the same configuration;
  kernels  (--profile) device time per kernel of one 8 x 1080p call, from torch.profiler, in a run of its own.
Each number is repeated --repeats times; min, median and max are reported.
"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from encode_bench import card, crowd, photo, stats  # noqa: E402


def profile(eng, frames, gpu):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile

    eng.encode_png(frames)
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.encode_png(frames)
    rows = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            rows[e.name] = rows.get(e.name, 0.0) + e.device_time_total / 1000.0
    top = sorted(rows.items(), key=lambda kv: -kv[1])[:20]
    print(json.dumps({"what": "kernels", "size": "1920x1080", "batch": len(frames),
                      "ms": {k[:60]: round(v, 3) for k, v in top}, "gpu": gpu}), flush=True)


def main():
    import cv2

    from smap_b200 import schema
    from smap_b200.engine import Engine
    from smap_b200.run_inference import run

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cli_frames", type=int, default=32)
    ap.add_argument("--skip_cli", action="store_true", help="only the encode and cv2 legs")
    ap.add_argument("--profile", action="store_true", help="only the per-kernel device times")
    a = ap.parse_args()
    gpu = card()
    eng = Engine(0, max_batch=8)
    B = 8
    if a.profile:
        profile(eng, [torch.from_numpy(photo(1080, 1920, s)).cuda() for s in range(B)], gpu)
        eng.close()
        return
    for h, w in ((1080, 1920), (3024, 4032)):
        frames = [torch.from_numpy(photo(h, w, s)).cuda() for s in range(B)]
        host = [f.cpu().numpy() for f in frames]
        for overlay in (False, True):
            extra = crowd(B, h, w, 1) if overlay else (None, None)
            eng.encode_png(frames, *extra)  # warm-up: workspace growth, module load
            iters = 10 if h == 1080 else 3
            rates = []
            for _ in range(a.repeats):
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(iters):
                    eng.encode_png(frames, *extra)
                rates.append(iters * B / (time.perf_counter() - t))
            print(json.dumps({"what": "encode", "size": "%dx%d" % (w, h), "batch": B, "overlay": overlay,
                              "frames_per_s": stats(rates), "gpu": gpu}), flush=True)
        for threads in (1, 8):
            cv2.setNumThreads(1)
            rates = []
            for _ in range(a.repeats):
                t = time.perf_counter()
                with ThreadPoolExecutor(threads) as ex:
                    list(ex.map(lambda f: cv2.imencode(".png", f), host))
                rates.append(B / (time.perf_counter() - t))
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
        for fmt in ("jpg", "png"):
            kw = dict(batch_size=8, vis_dir=os.path.join(tmp, "vis_" + fmt), vis_format=fmt)
            run(sd, data, os.path.join(tmp, "r.json"), **kw)  # warm-up
            rates = []
            for _ in range(a.repeats):
                t = time.perf_counter()
                run(sd, data, os.path.join(tmp, "r.json"), **kw)
                rates.append(a.cli_frames / (time.perf_counter() - t))
            print(json.dumps({"what": "cli", "vis_format": fmt, "frames": a.cli_frames, "frames_per_s": stats(rates),
                              "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
