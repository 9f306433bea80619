"""GPU: regenerate the committed tile-shape table (smap_b200/tiles/h100.tsv).  Builds the execution plans of the batch sizes
the bench, smoke() and the tests use at 832x512 with the autotuner on, and dumps what it measured.
    python tools/make_tile_table.py out/h100.tsv [batch ...]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SMAPB_NO_TILE_TABLE"] = "1"  # measure from scratch
import torch

from smap_b200 import schema
from smap_b200.engine import Engine, get_tile_table

out = sys.argv[1] if len(sys.argv) > 1 else "out/h100.tsv"
batches = [int(v) for v in sys.argv[2:]] or [8, 1, 2, 4]
sd = schema.make_state_dict(0, "identity")
for B in batches:
    e = Engine(0, max_batch=B, in_h=512, in_w=832)
    e.load_state_dict(sd)
    x = schema.make_input(B, 512, 832, seed=1).cuda()
    e.forward(x)
    torch.cuda.synchronize()
    e.close()
txt = get_tile_table()
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
with open(out, "w") as f:
    f.write("# layer geometry -> BLOCK_N, cta_group; measured on %s by tools/make_tile_table.py (batches %s)\n"
            % (torch.cuda.get_device_name(0), batches))
    f.write(txt)
print("%d entries -> %s" % (txt.count("\n"), out))
from collections import Counter
print(Counter(tuple(l.split("\t")[1:]) for l in txt.strip().split("\n")))
