"""CPU restatement of the 3D panel smapb_encode_jpeg_ex(SMAPB_ENCODE_VIEW3D) draws beside each frame
(smap_b200/csrc/view3d.cu, rules in include/smap_b200.h): render_view3d(frame, record, scale_row) -> the composite the
encoder compresses, so that jpeg_encode_numpy.encode(render_view3d(...)) equals the GPU output byte for byte.

The panel shows pred3d from lib/visualize/vis.py's viewpoint (azim -90, elev -45): screen right is +X, screen up is
(Z - Y) / sqrt(2), and the viewer looks along +(Y + Z).  Unlike vis.py the projection is orthographic with one scale on
both axes.  The fit is float64 with every operation rounded on its own, as numpy evaluates it (no fused multiply-add).
"""
import numpy as np

from oracle.render_numpy import COORD_MAX, PAIRS, PALETTE, limb_mask, render

S = 0.7071067811865476  # the float64 nearest sqrt(1/2)
MAX_COORD = 1e15
GREY = (160, 160, 160)
WHITE = (255, 255, 255)
# the fit box's edges between corners c whose bits 0, 1, 2 pick the maximum of X, Y, Z: 4 along X, 4 along Y, 4 along Z
BOX_EDGES = [(0, 1), (2, 3), (4, 5), (6, 7), (0, 2), (1, 3), (4, 6), (5, 7), (0, 4), (1, 5), (2, 6), (3, 7)]


def placed(record):
    """-> bool [n, 15] for the n = count rows: score > 0 and X, Y, Z finite with |.| <= 1e15."""
    n = min(max(int(record["count"]), 0), record["pred3d"].shape[0])
    q = np.asarray(record["pred3d"][:n], np.float64)
    with np.errstate(invalid="ignore"):
        return (q[..., 3] > 0) & (np.abs(q[..., :3]) <= MAX_COORD).all(-1)


def drawn_limbs(record):
    """-> [(row, limb index)] of the limbs whose joints are both placed, in (row, limb) order."""
    ok = placed(record)
    return [(p, k) for p in range(len(ok)) for k, (i, j) in enumerate(PAIRS) if ok[p, i] and ok[p, j]]


def fit(record, P):
    """-> (project, box) for a P x P panel, or None when no limb is drawn.  project(X, Y, Z) -> (x, y) pixel; box: the
    12 edges of the fit set's box as pairs of pixels, in paint order."""
    limbs = drawn_limbs(record)
    if not limbs:
        return None
    pose = record["pred3d"]
    pts = np.array([pose[p, j, :3] for p, k in limbs for j in PAIRS[k]], np.float64)
    X, Y, Z = pts[:, 0], pts[:, 1], pts[:, 2]
    a, b = X, (Z - Y) * S
    amin, amax, bmin, bmax = a.min(), a.max(), b.min(), b.max()
    m = P // 20
    avail = float(P - 1 - 2 * m)
    ea, eb = amax - amin, bmax - bmin
    span = max(ea, eb)
    with np.errstate(over="ignore"):
        k = avail / span if span > 0 and avail > 0 else np.float64(0)
        if not np.isfinite(k):
            k = np.float64(0)
        ox = m + (avail - ea * k) / 2
        oy = m + (avail - eb * k) / 2

    def project(x, y, z):
        with np.errstate(over="ignore"):
            u = ox + (np.float64(x) - amin) * k
            v = oy + (bmax - (np.float64(z) - np.float64(y)) * S) * k
        return tuple(int(np.clip(np.rint(t), -COORD_MAX, COORD_MAX)) for t in (u, v))

    lo, hi = (X.min(), Y.min(), Z.min()), (X.max(), Y.max(), Z.max())
    corner = [project(*[(hi if c >> i & 1 else lo)[i] for i in range(3)]) for c in range(8)]
    return project, [(corner[c0], corner[c1]) for c0, c1 in BOX_EDGES]


def elements(record, P):
    """-> the panel's elements in paint order: (a, b, BGR colour), a and b pixels."""
    f = fit(record, P)
    if f is None:
        return []
    project, box = f
    pose = record["pred3d"]
    out = [(a, b, GREY) for a, b in box]

    def depth(pk):
        p, k = pk
        i, j = PAIRS[k]
        return (pose[p, i, 1] + pose[p, i, 2]) + (pose[p, j, 1] + pose[p, j, 2])

    for p, k in sorted(drawn_limbs(record), key=lambda pk: (-depth(pk), pk)):
        i, j = PAIRS[k]
        out.append((project(*pose[p, i, :3]), project(*pose[p, j, :3]), PALETTE[p % len(PALETTE)]))
    return out


def panel(record, P):
    """One RECORD_DTYPE record -> uint8 BGR [P, P, 3]: its 3D skeletons on white, the fit box under them."""
    out = np.full((P, P, 3), 255, np.uint8)
    r = max(1, P // 400)
    for a, b, colour in elements(record, P):
        x0, x1 = max(0, min(a[0], b[0]) - r), min(P - 1, max(a[0], b[0]) + r)
        y0, y1 = max(0, min(a[1], b[1]) - r), min(P - 1, max(a[1], b[1]) + r)
        if x0 > x1 or y0 > y1:
            continue
        ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.int64)
        out[y0:y1 + 1, x0:x1 + 1][limb_mask(xs, ys, a, b, r)] = colour
    return out


def render_view3d(frame, record, scale_row):
    """uint8 BGR [h, w, 3] -> the h x (w + h) composite: the frame with its overlay (render_numpy.render), then the panel."""
    return np.hstack([render(frame, record, scale_row), panel(record, frame.shape[0])])
