"""Golden fixture for tests/test_shims_schema_cpu.py: the state-dict schema and seeded random init of the UNMODIFIED
reference modules model.smap.SMAP (torch.manual_seed(0)) and model.refinenet.RefineNet (torch.manual_seed(3)).

  reference_init.json.gz : per module, one [key, shape, dtype, first 8 hex digits of the sha256 of the tensor bytes]
                           row per state-dict entry, in state-dict order.

Run where the reference tree exists:  python tests/golden/make_golden_init.py REFERENCE_ROOT
"""
import gzip
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from test_shims_schema_cpu import _cfg, _import_from  # noqa: E402


def schema_rows(sd):
    return [[k, list(v.shape), str(v.dtype), hashlib.sha256(v.contiguous().numpy().tobytes()).hexdigest()[:8]]
            for k, v in sd.items()]


def main(ref):
    ref_smap, ref_refine = _import_from(ref, ["model.smap", "model.refinenet"])
    torch.manual_seed(0)
    smap = schema_rows(ref_smap.SMAP(_cfg()).state_dict())
    torch.manual_seed(3)
    refine = schema_rows(ref_refine.RefineNet().state_dict())
    raw = json.dumps({"smap_seed0": smap, "refinenet_seed3": refine}, separators=(",", ":")).encode()
    with gzip.GzipFile(os.path.join(HERE, "reference_init.json.gz"), "wb", mtime=0) as f:
        f.write(raw)


if __name__ == "__main__":
    main(sys.argv[1])
