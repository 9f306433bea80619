"""CPU restatement of the skeleton overlay smapb_encode_jpeg draws before encoding (smap_b200/csrc/jpeg_enc.cu,
include/smap_b200.h): render(frame, record, scale_row) -> the frame the encoder compresses, so that
jpeg_encode_numpy.encode(render(...)) equals the GPU output byte for byte.

Painter's order: persons in row order, each one's 14 limbs, then its 15 joints, later elements over earlier ones, opaque.
Every coverage test is exact integer arithmetic (int64), so there is nothing to round differently.
"""
import numpy as np

PAIRS = [[0, 1], [0, 2], [0, 9], [9, 10], [10, 11], [0, 3], [3, 4], [4, 5], [2, 12], [12, 13], [13, 14], [2, 6], [6, 7], [7, 8]]
PALETTE = [(0, 0, 255), (0, 255, 0), (255, 0, 0), (0, 255, 255), (0, 0, 0), (255, 0, 255)]  # BGR limb colour of person p % 6
JOINT = (255, 255, 255)
COORD_MAX = 32768


def radii(h, w):
    """-> (limb half-width r, joint radius R) of an h x w frame."""
    m = min(h, w)
    return max(1, m // 400), max(2, m // 200)


def letterbox(scale_row):
    """Scale row (scale, img_w, img_h, net_w, net_h, ...) -> (scale, pad_l, pad_t): the integer letterbox pre-processing
    applied (smap_b200/csrc/preprocess.cu, make_resize_plan)."""
    s, W, H, nw, nh = (float(v) for v in scale_row[:5])
    dw, dh = int(np.rint(W * s)), int(np.rint(H * s))
    pad_l = pad_t = 0
    if dw < nw:
        pad_l = (int(nw) - dw) // 2
    elif dh < nh:
        pad_t = (int(nh) - dh) // 2
    return s, pad_l, pad_t


def joints(record, scale_row):
    """-> list per person (row < count) of 15 (x, y) frame pixels, None for joints that are not drawn."""
    s, pad_l, pad_t = letterbox(scale_row)
    out = []
    for p in range(int(record["count"])):
        row = []
        for x, y, _, score in record["pred2d"][p]:
            if not (score > 0) or not (np.isfinite(x) and np.isfinite(y)):
                row.append(None)
                continue
            fx = np.clip(np.rint((float(x) - pad_l) / s), -COORD_MAX, COORD_MAX)
            fy = np.clip(np.rint((float(y) - pad_t) / s), -COORD_MAX, COORD_MAX)
            row.append((int(fx), int(fy)))
        out.append(row)
    return out


def limb_mask(xs, ys, a, b, r):
    """Clamped-projection test of the pixels (xs, ys) (int64 grids) against the limb a-b of half-width r."""
    vx, vy = b[0] - a[0], b[1] - a[1]
    px, py = xs - a[0], ys - a[1]
    dot, len2 = px * vx + py * vy, vx * vx + vy * vy
    cross = px * vy - py * vx
    small = np.abs(cross) <= (1 << 31)  # beyond it cross^2 > r^2 |b-a|^2 anyway, and the square would overflow
    mid = small & (np.where(small, cross, 0) ** 2 <= r * r * len2)
    return np.where(dot <= 0, px * px + py * py <= r * r,
                    np.where(dot >= len2, (xs - b[0]) ** 2 + (ys - b[1]) ** 2 <= r * r, mid))


def render(frame, record, scale_row):
    """uint8 BGR [H,W,3], one RECORD_DTYPE record and its scale row -> a new uint8 BGR frame with the skeletons drawn."""
    out = np.array(frame, np.uint8, copy=True)
    H, W = out.shape[:2]
    r, R = radii(H, W)
    for p, pts in enumerate(joints(record, scale_row)):
        elems = [(pts[i], pts[j], r, PALETTE[p % len(PALETTE)]) for i, j in PAIRS if pts[i] is not None and pts[j] is not None]
        elems += [(q, q, R, JOINT) for q in pts if q is not None]
        for a, b, rad, colour in elems:
            x0, x1 = max(0, min(a[0], b[0]) - rad), min(W - 1, max(a[0], b[0]) + rad)
            y0, y1 = max(0, min(a[1], b[1]) - rad), min(H - 1, max(a[1], b[1]) + rad)
            if x0 > x1 or y0 > y1:
                continue
            ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.int64)
            out[y0:y1 + 1, x0:x1 + 1][limb_mask(xs, ys, a, b, rad)] = colour
    return out
