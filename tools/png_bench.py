"""PNG decoding on the GPU against cv2 (tools only).

Seeded in-memory 1920x1080 and 4032x3024 frames (tests/golden/png_corpus.large_frames: gradients with mild noise, written
alternately by cv2.imencode with its defaults and by zlib level 6 over Paeth rows) are decoded
  1. by Engine.decode_png in batches of --batch (host chunk walk, upload, every phase, status read-back: the whole call),
  2. by cv2.imdecode on one thread, and on a pool of all host cores,
in images/s and Mpixel/s, with the share of kernel time per phase (torch.profiler, one call), the block finder's
candidates and false positives and the blocks per image.  Then the run_inference loop from file bytes to skeleton records
(decode, preprocess, infer_device, records to the host) is timed in bf16x3 and fp16 with each decoder (cv2 on one thread
is what the CLI did before).  The GPU's name, power limit and SM clock are read in the same call.

--single-block instead times one 1920x1080 frame stored as a single dynamic block of literals (as fpnge-style writers
store a frame): a block of millions of symbols is past the count pass's symbol cap, so the chain walk and the write pass
each decode it on one thread.  The same frame written by cv2.imencode (hundreds of blocks) is timed beside it.

    python tools/png_bench.py [--batch 8] [--rounds 5] [--json out/png_bench.json]
    python tools/png_bench.py --single-block [--rounds 5] [--json out/png_single_block.json]
"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from decode_bench import cv2_decode, gpu_info, sm_clock, timed  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

from deflate_writer import one_block_zlib  # noqa: E402
from png_corpus import large_frames, scanlines, write_png  # noqa: E402
from smap_b200 import schema  # noqa: E402
from smap_b200.engine import RECORD_BYTES, Engine  # noqa: E402

PHASES = ("gather_kernel", "find_kernel", "count_kernel", "chain_kernel", "write_kernel", "resolve_kernel", "unfilter_kernel",
          "colour_kernel")


def phase_shares(eng, files):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.decode_png(files)
        torch.cuda.synchronize()
    by = dict.fromkeys(PHASES, 0.0)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        for p in PHASES:
            if p in e.key:
                by[p] += t
    tot = sum(by.values())
    return {"kernel_ms": round(tot / 1e3, 3), **{p: round(v / tot, 3) for p, v in by.items()}} if tot else None


def single_block(a):
    from jpeg_corpus import content
    from png_corpus import cv2_png

    name, power = gpu_info()
    im = content("smooth", 1080, 1920, np.random.default_rng(1))
    s = np.ascontiguousarray(im[..., ::-1])
    one = write_png(s, 2, 8, z=one_block_zlib(scanlines(s, 2, 8, 0, lambda r: 4)))
    out = {"gpu": name, "power_limit": power, "frame": "1920x1080", "rounds": a.rounds}
    eng = Engine(0, max_batch=1)
    for key, f in (("one_dynamic_block", one), ("cv2_imencode", cv2_png(im))):
        (g,) = eng.decode_png([f])
        assert g is not None and np.array_equal(g.cpu().numpy(), cv2_decode(f)), key
        row = {"mbytes": round(len(f) / 1e6, 3), "finder": eng.png_stats()}
        for arm, fn in (("gpu_ms", lambda: eng.decode_png([f])), ("cv2_1_thread_ms", lambda: cv2_decode(f))):
            row[arm] = round(1e3 * timed(fn, a.rounds), 2)
        row["sm_clock_mhz"] = sm_clock()
        row["phase_share_of_kernel_time"] = phase_shares(eng, [f])
        out[key] = row
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default="")
    ap.add_argument("--single-block", action="store_true")
    a = ap.parse_args()
    if a.single_block:
        out = single_block(a)
        print(json.dumps(out))
        if a.json:
            os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
            with open(a.json, "w") as f:
                f.write(json.dumps(out) + "\n")
        return
    B = a.batch
    cores = os.cpu_count() or 1
    pool = ThreadPoolExecutor(cores)
    name, power = gpu_info()
    out = {"gpu": name, "power_limit": power, "host_cores": cores, "batch": B, "decode": {}, "cli": {}}
    eng = Engine(0, max_batch=B)
    corpora = {"%dx%d" % (w, h): [b for _, b in large_frames(n=B, sizes=((h, w),))] for h, w in ((1080, 1920), (3024, 4032))}
    for key, files in corpora.items():
        mpx = sum(int(np.prod(cv2_decode(f).shape[:2])) for f in files) / 1e6
        got = eng.decode_png(files)
        assert all(g is not None and np.array_equal(g.cpu().numpy(), cv2_decode(f)) for g, f in zip(got, files))
        st = eng.png_stats()
        row = {"mbytes_per_image": round(sum(map(len, files)) / len(files) / 1e6, 3),
               "blocks_per_image": round((st["confirmed"] + st["serial"]) / len(files), 1), "finder": st}
        for arm, fn in (("gpu", lambda: eng.decode_png(files)),
                        ("cv2_1_thread", lambda: [cv2_decode(f) for f in files]),
                        ("cv2_%d_threads" % cores, lambda: list(pool.map(cv2_decode, files)))):
            t = timed(fn, a.rounds)
            row[arm] = {"images_per_s": round(len(files) / t, 1), "mpixel_per_s": round(mpx / t, 1)}
            if arm == "gpu":
                row["sm_clock_mhz_after_gpu_arm"] = sm_clock()
        row["phase_share_of_kernel_time"] = phase_shares(eng, files)
        out["decode"][key] = row
    # the CLI loop: bytes -> records, 4 batches of 1920x1080 frames per round
    files = corpora["1920x1080"] * 4
    host = torch.empty(B, RECORD_BYTES, dtype=torch.uint8).pin_memory()
    sd = schema.make_state_dict(0, "identity")
    for prec in ("bf16x3", "fp16"):
        eng.load_state_dict(sd, prec)

        def loop(gpu_decode):
            for lo in range(0, len(files), B):
                chunk = files[lo:lo + B]
                frames = eng.decode_png(chunk) if gpu_decode else [torch.from_numpy(cv2_decode(f)) for f in chunk]
                imgs, scales = eng.preprocess(frames)
                rec = eng.infer_device(imgs, scales.to(imgs.device))
                host[:len(chunk)].copy_(rec)
                torch.cuda.current_stream().synchronize()

        row = {}
        for arm, flag in (("gpu_decode", True), ("cv2_1_thread", False)):
            t = timed(lambda: loop(flag), a.rounds)
            row[arm] = {"frames_per_s": round(len(files) / t, 1)}
        out["cli"][prec] = row
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
