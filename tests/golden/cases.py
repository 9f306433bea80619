"""Seeded input generators shared by make_golden.py (which feeds them to the reference) and the tests
(which feed them to the oracle / the CUDA path).  Pure numpy, no reference and no oracle code."""
import numpy as np

GEOMS = [(1920, 1080), (640, 480), (1000, 1500), (832, 512)]
N_LIFT_CASES = 24


def lift_case_inputs(ci):
    """-> bodies float32 [P,15,4] (heat-map px, as dapalib.connect returns), det_d [14,128,208],
    root_d [128,208], (img_w, img_h)."""
    rng = np.random.default_rng(100 + ci)
    P = int(rng.integers(0, 9))
    b = np.zeros((P, 15, 4), np.float32)
    b[:, :, 0] = rng.uniform(0.5, 207.4, (P, 15))
    b[:, :, 1] = rng.uniform(0.5, 127.4, (P, 15))
    b[:, :, 3] = rng.uniform(0.2, 1, (P, 15)) * (rng.uniform(size=(P, 15)) > 0.25)
    if P and ci % 5 == 0:
        b[0, 2, 3] = 0  # root missing -> dropped by register_pred
    b[b[:, :, 3] == 0] = 0
    det_d = rng.normal(0, 20, (14, 128, 208)).astype(np.float32)
    root_d = rng.uniform(1, 9, (128, 208)).astype(np.float32)
    return b, det_d, root_d, GEOMS[ci % 4]


def refine_state_dict(seed=7):
    """Seeded RefineNet weights with non-trivial BatchNorm statistics (pure generator: keys/shapes follow
    model/refinenet.py:8-17).  -> {key: float32 ndarray}"""
    rng = np.random.default_rng(seed)
    layers = [(75, 160), (160, 256), (256, 256), (256, 128)]
    sd = {}
    for i, (k, n) in enumerate(layers, start=1):
        p = "block.layer%d." % i
        sd[p + "0.weight"] = (rng.uniform(-1, 1, (n, k)) / np.sqrt(k)).astype(np.float32)
        sd[p + "0.bias"] = rng.uniform(-0.1, 0.1, n).astype(np.float32)
        sd[p + "1.weight"] = rng.uniform(0.5, 1.5, n).astype(np.float32)
        sd[p + "1.bias"] = rng.normal(0, 0.2, n).astype(np.float32)
        sd[p + "1.running_mean"] = rng.normal(0, 0.3, n).astype(np.float32)
        sd[p + "1.running_var"] = rng.uniform(0.5, 2.0, n).astype(np.float32)
        sd[p + "1.num_batches_tracked"] = np.asarray(100, np.int64)
    sd["block.layer5.weight"] = (rng.uniform(-1, 1, (45, 128)) / np.sqrt(128)).astype(np.float32)
    sd["block.layer5.bias"] = rng.uniform(-0.1, 0.1, 45).astype(np.float32)
    return sd


PRE_GEOMS = [(1920, 1080), (640, 480), (1000, 1500), (832, 512), (1664, 1024), (1280, 720), (333, 517), (2592, 1944),
             (500, 300), (831, 511), (1665, 1025), (100, 60), (2048, 1024), (416, 256), (3840, 2160), (517, 333)]


def preprocess_case_image(ci):
    """Seeded uint8 BGR test image [H,W,3] for geometry PRE_GEOMS[ci]: smooth low-frequency structure (so that the
    bilinear weights matter) plus full-range noise (so that every rounding case occurs)."""
    W, H = PRE_GEOMS[ci]
    rng = np.random.default_rng(500 + ci)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    base = 127 + 90 * np.sin(xx / (7 + ci))[:, :, None] * np.cos(yy / (11 + ci))[:, :, None] * np.array([1, 0.7, -0.8], np.float32)
    img = base + rng.normal(0, 40, (H, W, 3))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


# Network input sizes (net_w, net_h) the resize sweep runs at: the default, config 5, and the edge sizes of the plan
# tests (levels one row high, one column wide, the smallest tiled input).
RESIZE_NETS = [(832, 512), (1024, 1024), (96, 64), (992, 32), (32, 1024)]
RESIZE_KINDS = ("noise", "check", "flat")


def resize_geoms(net_w=832, net_h=512, n_random=None, seed=21):
    """Source geometries (W, H) that reach every regime of cv2.resize(img, (0,0), fx=s, fy=s), s = min(net_w/W, net_h/H),
    for a net_w x net_h input.  Includes geometries cv2 refuses (a resized side rounds to 0).
      * exact 1/2 scale with every parity of W mod 4 (H = 2 net_h) and of H mod 4 (W = 2 net_w): rint(W / 2) rounds up
        at W = 3 (mod 4), so the last column's 2x2 INTER_AREA window is cut by the image edge (likewise rows);
      * identity (s = 1 with nothing to resize) and near-identity;
      * up-scaling from 1-, 2- and few-pixel images;
      * extreme aspect ratios: a side resized to one pixel, or to rint(0.5) = 0 (refused);
      * exact 1/3 and 1/4 scales;
      * seeded random sizes (n_random; default: enough for more than 256 accepted geometries at 832x512, past the
        library's per-handle plan cache)."""
    hw, hh = 2 * net_w, 2 * net_h

    def sides(n):  # runs of 4 or more consecutive sides (every residue mod 4) at the small, middle and top end
        return sorted(set(range(2, 18)) | set(range(n // 2 - 2, n // 2 + 2)) | set(range(3 * n // 4 - 2, 3 * n // 4 + 2))
                      | set(range(n - 7, n + 1)))

    g = [(w, hh) for w in sides(hw)] + [(hw, h) for h in sides(hh)]
    if (net_w, net_h) == (832, 512):  # odd crops of a 1024-high photo (last column cut), and neighbours just off 1/2 scale
        g += [(767, 1024), (1363, 1024), (1663, 1023), (1665, 1024), (1664, 1025)]
    g += [(net_w, net_h), (net_w - 1, net_h), (net_w + 1, net_h + 1), (net_w - 1, net_h - 1)]
    g += [(1, 1), (1, 2), (2, 1), (2, 2), (5, 7), (17, 9), (1, 300), (5, 1), (net_w, 1), (1, net_h)]
    g += [(16384, 16), (17, 16384), (16, 16384), (16384, 9), (2, 16384), (1, hh), (5000, 40), (40, 5000)]
    g += [(3 * net_w, 3 * net_h), (3 * net_w, 3 * net_h - 1), (3 * net_w - 1, 3 * net_h), (4 * net_w, 4 * net_h),
          (4 * net_w + 1, 4 * net_h), (4 * net_w, 4 * net_h - 3), (3 * net_w + 2, 2 * net_h + 1)]
    g = [(w, h) for (w, h) in dict.fromkeys(g) if 1 <= w <= 16384 and 1 <= h <= 16384]
    if n_random is None:
        n_random = max(0, 280 - len(g))
    rng = np.random.default_rng(seed)
    while n_random > 0:
        w, h = int(rng.integers(1, 2600)), int(rng.integers(1, 2000))
        if (w, h) not in g:
            g.append((w, h))
            n_random -= 1
    return g


def resize_refused(W, H, net_w=832, net_h=512):
    """cv2.resize raises !dsize.empty() where a resized side rounds (half to even) to 0."""
    s = min(net_w / W, net_h / H)
    return int(np.rint(W * s)) == 0 or int(np.rint(H * s)) == 0


def resize_image(kind, W, H, seed):
    """uint8 BGR [H,W,3]: full-range noise (odd 2x2 and 1x2 sums, so round-half-to-even occurs), a 0/255 checkerboard
    (neighbours differ by the whole range) or flat 255 (the saturation edge)."""
    if kind == "noise":
        return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "check":
        c = ((np.add.outer(np.arange(H), np.arange(W)) % 2) * 255).astype(np.uint8)
        return np.stack([c, 255 - c, c], 2)
    return np.full((H, W, 3), 255, np.uint8)


def cv2_preprocess(img, net_w=832, net_h=512):
    """The reference loader with cv2 itself (dataset/custom_dataset.py:42-68, 23-24; exps/stage3_root2/test.py:99-103):
    cv2.resize(img, (0,0), fx=s, fy=s), gray-128 letterbox to net_w x net_h, ToTensor + Normalize in float32.
    -> (float32 [3, net_h, net_w], scale dict).  Raises cv2.error where cv2 refuses the size."""
    import cv2

    H, W = img.shape[:2]
    s = min(net_w / W, net_h / H)
    r = cv2.resize(img, (0, 0), fx=s, fy=s)
    h, w = r.shape[:2]
    out = np.full((net_h, net_w, 3), 128, np.uint8)
    if w < net_w:
        assert h == net_h
        out[:, (net_w - w) // 2:(net_w - w) // 2 + w] = r
    else:
        assert w == net_w and h <= net_h
        out[(net_h - h) // 2:(net_h - h) // 2 + h] = r
    x = out.astype(np.float32) / np.float32(255)
    x = (x - np.array([0.406, 0.456, 0.485], np.float32)) / np.array([0.225, 0.224, 0.229], np.float32)  # BGR, config.py:34-35
    scale = {"scale": s, "img_width": W, "img_height": H, "net_width": net_w, "net_height": net_h,
             "f_x": W, "f_y": W, "cx": W / 2, "cy": H / 2}
    return np.ascontiguousarray(x.transpose(2, 0, 1)), scale


N_GT_CASES = 12


def lift_gt_case_inputs(ci):
    """Inputs of the GT-matching branch (exps/stage3_root2/test.py:73-95, test_util.py:21-39): the lift case `ci` plus
    ground-truth bodies float64 [G,15,11] = (x, y, Z, vis, X, Y, Z, f_x, f_y, cx, cy) in network-input pixels.
    GT roots are placed near predicted roots (inside and outside the 30 px gate), with exact ties, duplicates competing for
    one prediction, and unmatched persons."""
    b, det_d, root_d, (iw, ih) = lift_case_inputs(ci)
    rng = np.random.default_rng(900 + ci)
    P = len(b)
    G = int(rng.integers(1, 7))
    gt = np.zeros((G, 15, 11), np.float64)
    gt[:, :, 0] = rng.uniform(0, 832, (G, 15))
    gt[:, :, 1] = rng.uniform(0, 512, (G, 15))
    gt[:, :, 2] = rng.uniform(100, 800, (G, 15))
    gt[:, :, 3] = 2
    gt[:, :, 4:7] = rng.normal(0, 100, (G, 15, 3))
    gt[:, :, 7], gt[:, :, 8], gt[:, :, 9], gt[:, :, 10] = 1100.0 + ci, 1105.0 + ci, iw / 2 + 3.5, ih / 2 - 2.25
    for g in range(G):
        if P and rng.uniform() < 0.8:
            p = int(rng.integers(0, P))
            r = float(rng.choice([0.0, 3.0, 12.5, 29.0, 31.0, 45.0]))
            ang = rng.uniform(0, 2 * np.pi)
            gt[g, 2, 0] = np.float64(b[p, 2, 0]) * 4 + r * np.cos(ang)
            gt[g, 2, 1] = np.float64(b[p, 2, 1]) * 4 + r * np.sin(ang)
    if G >= 2 and P and ci % 3 == 0:  # two GT persons at EXACTLY the same distance from one prediction (tie order)
        p = 0
        gt[0, 2, :2] = (np.float64(b[p, 2, 0]) * 4 + 6.0, np.float64(b[p, 2, 1]) * 4)
        gt[1, 2, :2] = (np.float64(b[p, 2, 0]) * 4 - 6.0, np.float64(b[p, 2, 1]) * 4)
    return b, det_d, root_d, (iw, ih), gt
