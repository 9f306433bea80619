"""Opcode histogram of libsmap_b200.so (cuobjdump -sass): the SASS mnemonics that prove wgmma / TMA / mbarrier use:
HGMMA (wgmma.mma_async), WARPGROUP (wgmma fence / arrive), UTMALDG / UTMASTG (TMA tensor loads / stores), UBLKCP (1-D bulk
copy), SYNCS (mbarrier).   python tools/sass_histogram.py > out/sass_opcodes.txt"""
import collections
import os
import re
import subprocess
import sys

lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "smap_b200", "lib", "libsmap_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
total = collections.Counter()
per_kernel = collections.defaultdict(collections.Counter)
cur = None
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        continue
    m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]+)", line)
    if m:
        total[m.group(1)] += 1
        per_kernel[cur][m.group(1).split(".")[0]] += 1
KEYS = ("HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "FENCE", "HMMA", "IMMA")
print("opcode histogram of smap_b200/lib/libsmap_b200.so (cuobjdump -sass, sm_90a)")
for op, n in sorted(total.items(), key=lambda kv: -kv[1]):
    if op.startswith(KEYS):
        print("%8d  %s" % (n, op))
print("total SASS instructions: %d; HMMA/IMMA (mma.sync) instructions: %d" % (sum(total.values()), sum(n for o, n in total.items() if o.startswith(("HMMA", "IMMA")))))
print("\nper kernel (base mnemonics of the list above):")
for k, c in sorted(per_kernel.items()):
    sel = {o: n for o, n in c.items() if o.startswith(KEYS)}
    if sel:
        print("  %-60s %s" % (k[:60], " ".join("%s=%d" % kv for kv in sorted(sel.items()))))
sys.exit(0)
