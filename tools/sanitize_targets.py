"""Small-shape workload for compute-sanitizer (tools/gpu_sanitize.sh): every kernel family of the library once or twice -
tensor-core convs in every pipeline configuration (plain, residual ring, post-adds, K-concatenated pair, bilinear residual
via a whole forward, every tile width, thin heads), the elementwise kernels, NMS / PAF / grouping / lift, RefineNet, pre-processing -
at sizes the sanitizer's ~100x slowdown tolerates.  Not a test (no numerical check) and not a bench."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from smap_b200 import schema
from smap_b200.engine import Engine, scale_row
from smap_b200.synth import make_scene

which = sys.argv[1] if len(sys.argv) > 1 else "all"
eng = Engine(0, max_batch=2, in_h=64, in_w=96)
g = torch.Generator().manual_seed(1)
if which in ("all", "conv"):
    cases = [(1, 16, 24, 64, 64, 1, 1, False), (1, 16, 24, 64, 256, 1, 1, True), (2, 16, 26, 128, 128, 3, 1, False),
             (1, 16, 26, 128, 128, 3, 2, False), (2, 16, 26, 256, 64, 1, 1, False), (1, 16, 24, 256, 14, 3, 1, False),
             (3, 20, 26, 64, 64, 3, 1, False)]
    for tile in (None, "128", "64", "32"):
        if tile:
            os.environ["SMAPB_FORCE_TILE"] = tile
        for (B, H, W, Cin, Cout, k, s, res) in cases:
            x = torch.randn(B, H, W, Cin, generator=g).cuda()
            w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
            b = torch.randn(Cout, generator=g).cuda()
            Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
            r = torch.randn(B, Ho, Wo, Cout, generator=g).cuda() if res and Cout % 32 == 0 else None
            eng.conv_test(x, w, b, res=r, stride=s, relu=True, post1=r, post2=r)
    os.environ.pop("SMAPB_FORCE_TILE", None)
    torch.cuda.synchronize()
    print("convs done")
if which in ("all", "path"):
    eng.load_state_dict(schema.make_state_dict(0, "random"))
    x = schema.make_input(2, 64, 96, seed=3).cuda()
    hm, dd, rd = eng.forward(x)  # whole backbone plan at 64x96: stem, maxpool, 194 convs incl. fused pairs / bilinear residuals, heads
    torch.cuda.synchronize()
    print("backbone done", float(hm.abs().max()))
if which in ("all", "assoc"):
    e2 = Engine(0, max_batch=2, in_h=512, in_w=832)
    ss = [make_scene(5 + i, 6) for i in range(2)]
    hms = torch.from_numpy(np.stack([s["hms"] for s in ss])).cuda()
    rdm = torch.from_numpy(np.stack([s["root_d"] for s in ss])).cuda()
    ddm = torch.from_numpy(np.stack([s["det_d"] for s in ss])).cuda()
    peaks, scores = e2.extract(hms)
    bodies, counts = e2.connect(hms, rdm)
    sc = dict(scale=832 / 1920, img_width=1920, img_height=1080, net_width=832, net_height=512, f_x=1920.0, f_y=1920.0, cx=960.0, cy=540.0)
    scales = torch.from_numpy(np.stack([scale_row(sc)] * 2)).cuda()
    e2.lift(bodies, counts, ddm, rdm, scales)
    gt = torch.zeros(2, 4, 2, dtype=torch.float64).cuda() + 100.0
    e2.lift_gt(bodies, counts, ddm, rdm, scales, gt, torch.tensor([3, 2], dtype=torch.int32).cuda())
    e2.merge_scale(torch.randn(2, 43, 128, 208).cuda(), torch.randn(2, 43, 128, 208).cuda(), True)
    img = torch.randint(0, 255, (300, 500, 3), dtype=torch.uint8).cuda()
    e2.preprocess([img])
    torch.cuda.synchronize()
    e2.close()
    print("association / lift / preprocess done", counts.tolist())
eng.close()
