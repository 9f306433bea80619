"""GPU-box diagnostic: where does the grouping differ from the unmodified reference extension?"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from oracle import assoc, build_ref
from test_assoc_gpu import scenes, random_heatmaps, edge_cases, H, W

ref = build_ref.load_ref()
sets = {"scenes": scenes(range(40, 44))[:2], "random": random_heatmaps(5, B=2)}
ec = edge_cases()
for name in ("plateau_border_threshold", "saturated_127_peaks", "coincident_and_near", "empty"):
    sets[name] = (ec[name][None], np.random.default_rng(3).uniform(0.5, 3, (1, H, W)).astype(np.float32))
for name, (hms, rd) in sets.items():
    for b in range(hms.shape[0]):
        th = torch.from_numpy(hms[b]).cuda()
        rb = ref.connect(th, torch.from_numpy(rd[b]), 2, True).numpy()
        ob, peaks, scores = assoc.connect(hms[b], rd[b], return_all=True)
        if rb.size == 0 and len(ob) == 0:
            print(name, b, "both empty"); continue
        same = rb.shape == ob.shape and np.array_equal(rb, ob)
        print(name, b, "P=", len(ob), "equal" if same else "DIFF")
        if not same and rb.shape == ob.shape:
            d = np.argwhere((rb != ob).any(-1))
            print("  first diffs (person, joint):", d[:10].tolist(), "total", len(d))
            for (p, j) in d[:5]:
                print("   ref", rb[p, j], "ora", ob[p, j])
            # depth ties?
            root = peaks[2]; n = int(root[0, 0])
            dep = np.array([rd[b][int(root[i + 1, 1]), int(root[i + 1, 0])] for i in range(n)])
            u, c = np.unique(dep, return_counts=True)
            print("  depth ties:", (c > 1).sum(), "nan:", np.isnan(dep).sum())
            np.savez("out/diag_%s_%d.npz" % (name, b), hms=hms[b], rd=rd[b], ref=rb, ora=ob)
# division semantics of torch on CUDA
x = torch.randn(1 << 20, device="cuda") * 100
a = x / 255
print("torch cuda x/255 == true div:", torch.equal(a, torch.from_numpy((x.cpu().numpy() / np.float32(255)).astype(np.float32)).cuda()),
      " == x*(1f/255):", torch.equal(a, x * torch.tensor(np.float32(1) / np.float32(255), device="cuda")))
y = x.clone(); y /= 127
print("inplace /=127 == x*(1f/127):", torch.equal(y, x * torch.tensor(np.float32(1) / np.float32(127), device="cuda")),
      "== true:", torch.equal(y, torch.from_numpy((x.cpu().numpy() / np.float32(127)).astype(np.float32)).cuda()))
xc = x.cpu(); yc = xc.clone(); yc /= 255
print("cpu inplace /=255 == true:", np.array_equal(yc.numpy(), (xc.numpy() / np.float32(255)).astype(np.float32)))
