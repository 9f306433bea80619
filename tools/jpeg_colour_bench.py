"""JPEG decoding on the GPU against cv2 for the frames SMAPB_JPEG_COLOUR adds (tools only).

Seeded 1920x1080 and 4032x3024 frames (smooth content, q90; tests/golden/jpeg_colour.py's large_frames) of four kinds -
Pillow's CMYK 4:4:4, Pillow's CMYK 4:2:0 (factors on C), the same relabelled YCCK, and cv2's 4:1:1 - are decoded in
batches of --batch (two distinct frames per kind and size, repeated to fill the batch, which keeps the seeded set-up
short) by Engine.decode_jpeg_ex(colour=True) (host parse, upload, every phase, status read-back: the whole
call) and by cv2.imdecode on one thread and on a pool of all host cores, in images/s and Mpixel/s.  Every GPU output is
checked against cv2's first.  The GPU's name, power limit and SM clock are read in the same call.  Each row is printed
as it is measured; the last line is the whole result as JSON.

    python tools/jpeg_colour_bench.py [--batch 8] [--rounds 3] [--json out/jpeg_colour_bench.json]
"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from decode_bench import cv2_decode, gpu_info, sm_clock, timed  # noqa: E402  (also puts the repository on sys.path)
from jpeg_colour import LARGE_KINDS, large_frames  # noqa: E402
from smap_b200.engine import Engine  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    B = a.batch
    cores = os.cpu_count() or 1
    pool = ThreadPoolExecutor(cores)
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "host_cores": cores, "batch": B, "decode": {}}
    eng = Engine(0, max_batch=B)
    for kind in LARGE_KINDS:
        for seed, (h, w) in enumerate(((1080, 1920), (3024, 4032))):
            files = (large_frames(kind, h, w, 2, seed=100 + seed) * B)[:B]
            refs = [cv2_decode(f) for f in files]
            got = eng.decode_jpeg_ex(files, colour=True)
            assert all(g is not None and np.array_equal(g.cpu().numpy(), r) for g, r in zip(got, refs)), kind
            mpx = sum(int(np.prod(r.shape[:2])) for r in refs) / 1e6
            row = {"mbytes_per_image": round(sum(map(len, files)) / len(files) / 1e6, 3)}
            for arm, fn in (("gpu", lambda: eng.decode_jpeg_ex(files, colour=True)),
                            ("cv2_1_thread", lambda: [cv2_decode(f) for f in files]),
                            ("cv2_%d_threads" % cores, lambda: list(pool.map(cv2_decode, files)))):
                t = timed(fn, a.rounds)
                row[arm] = {"images_per_s": round(len(files) / t, 1), "mpixel_per_s": round(mpx / t, 1)}
                if arm == "gpu":
                    row["sm_clock_mhz_after_gpu_arm"] = sm_clock()
            out["decode"]["%s_%dx%d" % (kind, w, h)] = row
            print(kind, w, h, json.dumps(row), flush=True)
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
