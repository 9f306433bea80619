"""GPU: time every BLOCK_N tile shape on the layer geometries of the bench workload through smapb_conv_test and
check that all shapes produce the SAME BITS (tools only; not a bench value).  python tools/tile_probe.py [names...]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from smap_b200.engine import Engine

SHAPES = {
    # name: (B, H, W, Cin, Cout, k, stride, relu, res)
    "l1_c3": (8, 128, 208, 64, 256, 1, 1, True, True),
    "l1_c1": (8, 128, 208, 256, 64, 1, 1, True, False),
    "l1_c2": (8, 128, 208, 64, 64, 3, 1, True, False),
    "up4_1x1": (8, 128, 208, 256, 256, 1, 1, True, False),
    "l2_c3": (8, 64, 104, 128, 512, 1, 1, True, True),
    "l2_c2": (8, 64, 104, 128, 128, 3, 1, True, False),
    "l2_c1": (8, 64, 104, 512, 128, 1, 1, True, False),
    "l3_c3": (8, 32, 52, 256, 1024, 1, 1, True, True),
    "l3_c2": (8, 32, 52, 256, 256, 3, 1, True, False),
    "l3_c1": (8, 32, 52, 1024, 256, 1, 1, True, False),
    "l4_c2": (8, 16, 26, 512, 512, 3, 1, True, False),
    "l4_c3": (8, 16, 26, 512, 2048, 1, 1, True, True),
    "l4_c1": (8, 16, 26, 2048, 512, 1, 1, True, False),
}
TILES = ("128", "64", "32")
names = sys.argv[1:] or list(SHAPES)
eng = Engine(0, max_batch=1, in_h=64, in_w=96)
g = torch.Generator(device="cpu").manual_seed(5)
for n in names:
    B, H, W, Cin, Cout, k, s, relu, res = SHAPES[n]
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    Ho, Wo = H // s, W // s
    r = torch.randn(B, Ho, Wo, Cout, generator=g).cuda() if res else None
    flops = 2.0 * B * Ho * Wo * Cout * Cin * k * k
    base = None
    out = []
    for t in TILES:
        if Cout % int(t):
            continue
        os.environ["SMAPB_FORCE_TILE"] = t
        try:
            y, ms = eng.conv_test(x, w, b, res=r, stride=s, relu=relu, time_it=True)
        except Exception as e:  # noqa: BLE001
            out.append("%s: %s" % (t, str(e)[:60]))
            continue
        torch.cuda.synchronize()
        if base is None:
            base = y
        same = torch.equal(y, base)
        out.append("%s %.3f ms %.0f TF/s %s" % (t, ms, flops / ms * 1e-9, "same-bits" if same else "DIFF %.2e" % (y - base).abs().max().item()))
    print("%-8s " % n + " | ".join(out), flush=True)
