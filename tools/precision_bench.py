"""Speed and accuracy of the three precisions side by side (tools only).

bench.py's workload - 8 x 832x512 frames per step, two handles with their own streams, CUDA-graph replay, device-resident
inputs - run for bf16x3, fp16 and bf16 alternately in one process, --rounds times, so that clock and neighbour drift hit
every mode alike.  Reports per mode the median frames/s over the rounds, the conv kernel ms per step (per-launch CUDA events,
profile_begin / profile_end, one handle, eager), the GPU's name, power limit and median SM clock, and the accuracy of the
backbone against the fp32 oracle (832x512 B=2, random BN) next to cuDNN with TF32.

    python tools/precision_bench.py [--steps 30] [--rounds 5] [--json out/precision_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from smap_b200 import schema  # noqa: E402
from smap_b200.engine import RECORD_BYTES, Engine, scale_row  # noqa: E402

MODES = ("bf16x3", "fp16", "bf16")
B, H, W, NE, NROT = 8, 512, 832, 2, 4


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip()


def accuracy():
    from oracle import smap_torch

    sd = smap_torch.make_state_dict(0, "random")
    x = smap_torch.make_input(2, H, W, seed=1).cuda()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = smap_torch.smap_forward(sd_dev, x)
    torch.backends.cudnn.allow_tf32 = True
    tf32 = smap_torch.smap_forward(sd_dev, x)
    torch.backends.cudnn.allow_tf32 = False
    rel = lambda a, b: (a - b).abs().max().item() / b.abs().max().item()  # noqa: E731
    out = {"cudnn_tf32": [rel(a, b) for a, b in zip(tf32, ref)]}
    eng = Engine(0, max_batch=2, in_h=H, in_w=W)
    try:
        for m in MODES:
            eng.load_state_dict(sd, m)
            out[m] = [rel(a, b) for a, b in zip(eng.forward(x), ref)]
            out[m + "_saturated"] = eng.saturation_count(reset=True)
    finally:
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    sd = schema.make_state_dict(0, "identity")
    batches = [schema.make_input(B, H, W, seed=1 + r).to(dev) for r in range(NROT)]
    sc = dict(scale=W / 1920, img_width=1920, img_height=1080, net_width=W, net_height=H, f_x=1920.0, f_y=1920.0,
              cx=960.0, cy=540.0)
    scales = torch.from_numpy(np.stack([scale_row(sc)] * B)).to(dev)
    engines, outs = {}, {}
    for m in MODES:
        engines[m] = [Engine(0, max_batch=B, in_h=H, in_w=W, stream=torch.cuda.Stream(dev)) for _ in range(NE)]
        for e in engines[m]:
            e.load_state_dict(sd, m)
        outs[m] = [torch.empty(B, RECORD_BYTES, dtype=torch.uint8, device=dev) for _ in range(NE)]
    cur = torch.cuda.current_stream()

    def run(m, steps):
        for i in range(steps):
            engines[m][i % NE].infer_device(batches[i % NROT], scales, out=outs[m][i % NE])

    def timed(m):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(cur)
        for e in engines[m]:
            e.stream.wait_event(e0)
        run(m, a.steps)
        for e in engines[m]:
            cur.wait_stream(e.stream)
        e1.record(cur)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for m in MODES:  # eager runs, graph capture for every (handle, batch) pair, then warm-up
        run(m, 3 * NE * NROT)
        run(m, 4)
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    fps = {m: [] for m in MODES}
    for _ in range(a.rounds):
        for m in MODES:
            fps[m].append(B * a.steps / (timed(m) * 1e-3))
    sampler.stop_flag = True
    sampler.join(timeout=2)
    conv_ms = {}
    for m in MODES:
        e = engines[m][0]
        e.profile_begin()
        for i in range(5):
            e.infer_device(batches[i % NROT], scales, out=outs[m][0])
        prof = e.profile_end()
        conv_ms[m] = prof["conv"][0] / 5
    sat = {m: sum(e.saturation_count() for e in engines[m]) for m in MODES}
    for m in MODES:
        for e in engines[m]:
            e.close()
    acc = accuracy()
    name, power = gpu_info()
    clk = sampler.result()
    res = {"gpu": name, "power_limit": power, "sm_mhz_median": clk["sm_mhz"], "clock_reasons": clk["reasons"],
           "steps": a.steps, "rounds": a.rounds, "frames_per_step": B, "handles": NE,
           "modes": {m: {"frames_per_s_median": statistics.median(fps[m]), "frames_per_s": fps[m],
                         "ms_per_step_median": B * 1e3 / statistics.median(fps[m]), "conv_ms_per_step_eager": conv_ms[m],
                         "saturation_count": sat[m]} for m in MODES},
           "accuracy_832x512_b2_random": acc}
    print("%s, power limit %s, median SM clock %s MHz (%s)" % (name, power, clk["sm_mhz"], ",".join(clk["reasons"]) or "-"))
    print("%-7s %12s %12s %16s" % ("mode", "frames/s", "ms/step", "conv ms/step"))
    for m in MODES:
        r = res["modes"][m]
        print("%-7s %12.1f %12.2f %16.2f" % (m, r["frames_per_s_median"], r["ms_per_step_median"], r["conv_ms_per_step_eager"]))
    print("max|a-b|/max|ref| vs the fp32 oracle (832x512 B=2, random BN): hm2d detd rootd")
    for k in ("fp16", "bf16", "bf16x3", "cudnn_tf32"):
        print("  %-11s %s" % (k, "  ".join("%.2e" % v for v in acc[k])))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
