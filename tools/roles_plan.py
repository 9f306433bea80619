"""Where every conv launch of one whole-path step waits (tools only): per-role wait cycles of the warp-specialised conv kernel
collected INSIDE the plan (cache state and clocks of the real step, one handle, eager), grouped by layer geometry.
  SMAPB_ROLES_PLAN=out/roles_plan.csv python tools/roles_plan.py
Columns (fractions of the CTA's lifetime, both consumer warpgroups together): operands not landed (load bound), waiting
for the main-loop turn (the other warpgroup's main loop: tensor bound), time in epilogues, and within it epilogue inputs not
landed (ring) and the staging slot still being stored (store bound)."""
import collections
import csv
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from smap_b200 import schema
from smap_b200.engine import RECORD_BYTES, Engine, scale_row

COLS = ("wait_full", "wait_order", "epilogue", "wait_ring", "wait_stage")  # per consumer warpgroup (smapb_profile_end)
path = os.environ.setdefault("SMAPB_ROLES_PLAN", "out/roles_plan.csv")
B, H, W = 8, 512, 832
eng = Engine(0, max_batch=B, in_h=H, in_w=W)
eng.load_state_dict(schema.make_state_dict(0, "identity"))
xs = [schema.make_input(B, H, W, seed=1 + r).cuda() for r in range(2)]
sc = dict(scale=W / 1920, img_width=1920, img_height=1080, net_width=W, net_height=H, f_x=1920.0, f_y=1920.0, cx=960.0, cy=540.0)
scales = torch.from_numpy(np.stack([scale_row(sc)] * B)).cuda()
out = torch.empty(B, RECORD_BYTES, dtype=torch.uint8, device="cuda")
for i in range(4):
    eng.infer_device(xs[i % 2], scales, out=out)
torch.cuda.synchronize()
eng.profile_begin()
for i in range(3):
    eng.infer_device(xs[i % 2], scales, out=out)
eng.profile_end(path.replace(".csv", "_ops.csv"))
eng.close()

rows = list(csv.DictReader(open(path)))
ops = list(csv.DictReader(open(path.replace(".csv", "_ops.csv"))))
ms_by_desc = collections.defaultdict(float)
for r in ops:
    ms_by_desc[r["desc"]] += float(r["ms"]) / 3
agg = collections.OrderedDict()
for r in rows:
    desc = r["desc"]
    a = agg.setdefault(desc, collections.defaultdict(float))
    a["n"] += 1
    for k in ("total", "producer_wait_empty") + tuple("g%d_%s" % (g, c) for g in (0, 1) for c in COLS):
        a[k] += float(r[k])
print("%-62s %7s %6s | %5s %5s %5s | %5s %5s" % ("layer", "ms/step", "n", "full", "order", "epi", "ring", "stage"))
for desc, a in sorted(agg.items(), key=lambda kv: -ms_by_desc.get(kv[0], 0)):
    t = a["total"] or 1.0
    e = lambda c: 50.0 * (a["g0_" + c] + a["g1_" + c]) / t
    print("%-62s %7.3f %6d | %4.0f%% %4.0f%% %4.0f%% | %4.0f%% %4.0f%%" % (desc[:62], ms_by_desc.get(desc, 0), a["n"] / 3,
          e("wait_full"), e("wait_order"), e("epilogue"), e("wait_ring"), e("wait_stage")))
