"""Summarise a per-op CSV written by smapb_profile_end (bench.py --profile-csv)."""
import collections
import csv
import sys

path = sys.argv[1] if len(sys.argv) > 1 else "out/ops.csv"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
top = int(sys.argv[3]) if len(sys.argv) > 3 else 30
rows = list(csv.DictReader(open(path)))
agg = collections.OrderedDict()
for r in rows:
    a = agg.setdefault((r["kind"], r["desc"]), [0, 0.0, 0.0])
    a[0] += 1
    a[1] += float(r["ms"])
    a[2] += float(r["gflop"])
tot = sum(a[1] for a in agg.values())
print("total %.3f ms/step" % (tot / steps))
for (k, d), (n, ms, gf) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
    print("%8.3f ms/step  n=%3d  %7.1f TF/s  %s" % (ms / steps, n // steps, gf / ms if ms > 0 else 0, d))
