"""Golden fixture for tests/test_assoc_gpu.py: sha256 digests (with shapes and dtypes) of the peaks, pair scores and bodies
the UNMODIFIED reference extension (oracle/_ref/dapalib_ref*.so, oracle/build_ref.py) returns on the inputs of that test.

Run on a GPU with the reference extension built:  python tests/golden/make_golden_assoc_ref.py OUT.npz
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import build_ref  # noqa: E402
from test_assoc_gpu import reference_sets, scenes  # noqa: E402


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def put_bodies(g, prefix, t):
    a = t.numpy()
    g[prefix + "bodies"] = np.array(digest(t))
    g[prefix + "body_shape"] = np.array(a.shape, np.int64)
    g[prefix + "body_dtype"] = np.array(str(a.dtype))


def main(out):
    ref = build_ref.load_ref()
    assert ref is not None, "oracle/_ref/dapalib_ref*.so is not built"
    g = {}
    for s, (hms, rd) in enumerate(reference_sets()):
        th = torch.from_numpy(hms).cuda()
        for b in range(hms.shape[0]):
            pc, sc = ref.extract(th[b].contiguous())
            g["s%d_b%d_peaks" % (s, b)] = np.array([digest(pc[j]) for j in range(15)])
            g["s%d_b%d_peak_shapes" % (s, b)] = np.array([tuple(pc[j].shape) for j in range(15)], np.int64)
            g["s%d_b%d_peak_dtype" % (s, b)] = np.array(str(pc[0].numpy().dtype))
            g["s%d_b%d_scores" % (s, b)] = np.array([digest(sc[l]) for l in range(14)])
            g["s%d_b%d_score_shapes" % (s, b)] = np.array([tuple(sc[l].shape) for l in range(14)], np.int64)
            put_bodies(g, "s%d_b%d_" % (s, b), ref.connect(th[b].contiguous(), torch.from_numpy(rd[b]), 2, True))
    hms, rd, _ = scenes(range(50, 53))
    for b in range(3):
        put_bodies(g, "o%d_" % b, ref.connect(torch.from_numpy(hms[b]).cuda(), torch.from_numpy(rd[b]), 2, True))
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **g)
    print("%d arrays -> %s" % (len(g), out))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "assoc_ref.npz"))
