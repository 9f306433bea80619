"""JPEG decoding on the GPU against cv2 (tools only).

A seeded in-memory corpus of q90 4:2:0 frames written by cv2 (1920x1080 and 4032x3024; gradients with noise, i.e. a
photo-like entropy of roughly 1-2 bits per pixel) is decoded
  1. by Engine.decode_jpeg in batches of --batch (host parse, upload, every phase, status read-back: the whole call),
  2. by cv2.imdecode on one thread, and on a pool of all host cores,
in images/s and Mpixel/s.  The same q90 4:2:0 frames written progressive by cv2 (libjpeg's default 10-scan script) are
decoded by Engine.decode_jpeg_ex against cv2, with the share of kernel time that goes to the AC refinement scans (the
history masks, one warp per restart segment decoding against them, and the apply pass; these files have no restart
markers) from torch.profiler.  Then the run_inference loop from files on disk to skeleton records (decode, preprocess,
infer_device, records to the host) is timed in bf16x3 and fp16, its GPU arm through run_inference.read_frames (the CLI's
own routing: decode_jpeg, then decode_jpeg_ex for the progressive files) and its cv2 arm through cv2.imread on one thread
(what the CLI did before).  The GPU's name, power limit and SM clock are read in the same call.

    python tools/decode_bench.py [--batch 8] [--rounds 5] [--json out/decode_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from jpeg_corpus import content, cv2_jpeg  # noqa: E402
from jpeg_scans import cv2_progressive  # noqa: E402
from smap_b200 import schema  # noqa: E402
from smap_b200.engine import RECORD_BYTES, Engine  # noqa: E402
from smap_b200.run_inference import read_frames  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip()


def sm_clock():
    """SM clock (MHz) now, read right after a timed loop."""
    q = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return q.stdout.strip()


def make_corpus(h, w, n, seed, progressive=False):
    rng = np.random.default_rng(seed)
    enc = cv2_progressive if progressive else cv2_jpeg
    return [enc(content("smooth", h, w, rng), 90, "420") for _ in range(n)]


def refine_share(eng, files):
    """Share of the decode call's kernel time spent in the AC refinement kernels (acr_*, torch.profiler, one call)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.decode_jpeg_ex(files)
        torch.cuda.synchronize()
    tot = ref = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if "kernel" in e.key and "Memcpy" not in e.key and "Memset" not in e.key:
            tot += t
            if "acr_mask_kernel" in e.key or "acr_decode_kernel" in e.key or "acr_apply_kernel" in e.key:
                ref += t
    return round(ref / tot, 3) if tot else None


def cv2_decode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def timed(fn, rounds):
    """median seconds of fn() over rounds, after one warm-up call."""
    fn()
    ts = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    B = a.batch
    cores = os.cpu_count() or 1
    pool = ThreadPoolExecutor(cores)
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "host_cores": cores, "batch": B, "decode": {}, "cli": {}}
    eng = Engine(0, max_batch=B)
    corpora = {"1920x1080": make_corpus(1080, 1920, B, 1), "4032x3024": make_corpus(3024, 4032, B, 2)}
    for key, files in corpora.items():
        mpx = sum(int(np.prod(cv2_decode(f).shape[:2])) for f in files) / 1e6
        assert all(o is not None for o in eng.decode_jpeg(files))
        row = {"mbytes_per_image": round(sum(map(len, files)) / len(files) / 1e6, 3)}
        for arm, fn in (("gpu", lambda: eng.decode_jpeg(files)),
                        ("cv2_1_thread", lambda: [cv2_decode(f) for f in files]),
                        ("cv2_%d_threads" % cores, lambda: list(pool.map(cv2_decode, files)))):
            t = timed(fn, a.rounds)
            row[arm] = {"images_per_s": round(len(files) / t, 1), "mpixel_per_s": round(mpx / t, 1)}
        out["decode"][key] = row
    for key, (h, w, seed) in {"prog_1920x1080": (1080, 1920, 3), "prog_4032x3024": (3024, 4032, 4)}.items():
        files = make_corpus(h, w, B, seed, progressive=True)
        mpx = sum(int(np.prod(cv2_decode(f).shape[:2])) for f in files) / 1e6
        assert all(o is not None for o in eng.decode_jpeg_ex(files))
        row = {"mbytes_per_image": round(sum(map(len, files)) / len(files) / 1e6, 3)}
        for arm, fn in (("gpu", lambda: eng.decode_jpeg_ex(files)),
                        ("cv2_1_thread", lambda: [cv2_decode(f) for f in files]),
                        ("cv2_%d_threads" % cores, lambda: list(pool.map(cv2_decode, files)))):
            t = timed(fn, a.rounds)
            row[arm] = {"images_per_s": round(len(files) / t, 1), "mpixel_per_s": round(mpx / t, 1)}
        eng.decode_jpeg_ex(files)
        row["sm_clock_mhz_after_gpu_arm"] = sm_clock()
        row["ac_refine_share_of_kernel_time"] = refine_share(eng, files)
        out["decode"][key] = row
    # the CLI loop: files -> records, 4 batches of 1920x1080 frames per round
    tmp = tempfile.TemporaryDirectory()
    paths = {}
    for kind, fs in (("baseline", corpora["1920x1080"]), ("progressive", make_corpus(1080, 1920, B, 3, progressive=True))):
        paths[kind] = []
        for k, b in enumerate(fs * 4):
            p = os.path.join(tmp.name, "%s_%02d.jpg" % (kind, k))
            with open(p, "wb") as f:
                f.write(b)
            paths[kind].append(p)
    host = torch.empty(B, RECORD_BYTES, dtype=torch.uint8).pin_memory()
    sd = schema.make_state_dict(0, "identity")

    def imread(p):
        return cv2.imread(p, cv2.IMREAD_COLOR)

    for prec in ("bf16x3", "fp16"):
        eng.load_state_dict(sd, prec)

        def loop(gpu_decode, ps):
            for lo in range(0, len(ps), B):
                chunk = ps[lo:lo + B]
                frames = read_frames(eng, chunk, imread) if gpu_decode else [imread(p) for p in chunk]
                frames = [f if torch.is_tensor(f) else torch.from_numpy(f) for f in frames]
                imgs, scales = eng.preprocess(frames)
                rec = eng.infer_device(imgs, scales.to(imgs.device))
                host[:len(chunk)].copy_(rec)
                torch.cuda.current_stream().synchronize()

        row = {}
        for kind, prefix in (("baseline", ""), ("progressive", "progressive_")):
            for arm, flag in (("gpu_decode", True), ("cv2_1_thread", False)):
                t = timed(lambda: loop(flag, paths[kind]), a.rounds)
                row[prefix + arm] = {"frames_per_s": round(len(paths[kind]) / t, 1)}
        out["cli"][prec] = row
    tmp.cleanup()
    eng.close()
    pool.shutdown()
    line = json.dumps(out)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
