"""Adversarial association frames: [43, h, w] float32 heat maps with [h, w] root-depth maps (128 x 208 by default),
built so that each rule of the reference association (extensions/gpu/nmsBase.cu, gpu/bodyPartConnectorBase.cu,
association.cpp) is reached where a restatement could misread it.  Seeded and deterministic; numpy only, apart from
the breadth family, which reuses the frames the other association tests build (at 128 x 208) or their generators.

Every frame is (name, hms, rdepth, targets); `targets` names the rules the frame is built to reach.  tests/
test_assoc_adversary_cpu.py checks with the oracle that each family reaches them; tests/test_assoc_reference_gpu.py
runs the kernels, the oracle and the live reference extension on them.  `frames(h, w)` builds the same families at
another map size (tests/test_assoc_sizes_*.py): the near threshold, grids, borders, corners, offsets, sweeps, the cap
frames and the depth maps follow (h, w); a frame whose rule cannot be reached at a size is left out, and `LEFT_OUT`
names why.  At 128 x 208 the frames are byte-identical to the ones this module built before it took a size.

Families:
  nms    values at 0.2f and one ulp either side; 2-, 3- and 4-pixel plateaus; peaks on rows / columns 1 and h-2 / w-2
         next to large border values; centroid windows clipped by every edge and corner; windows holding zeros,
         negatives, NaN, denormals (and +-inf and overflowing values in non-root planes); 127, 128 and 300 peaks in one
         plane; all 15 planes saturated.
  paf    coincident candidates (norm 0); integer offsets 0 ... 200 along x, y and the diagonal (every sample count
         n = 5 ... 25); direction sweeps whose samples land on k + 0.5; projections at 0.05f and one ulp either side;
         19 of 20 and 24 of 25 samples passing; distances just below and above the near threshold and around 1e-6;
         NaN and +-inf in the PAF planes.
  group  equal pair scores (first index wins, also across lanes); competition decided by the `used` flags in both
         depth orders; pair scores at exactly 0 and just above after the distance penalty; chains cut by a missing
         joint; 127 persons; root-depth key sets with ties, +-0, NaN, +-inf and negative depths.
  breadth  32 random_heatmaps seeds, 32 make_scene seeds, the crowded frames and the edge cases of the other tests.

Safety (the reference has no shape checks and indexes the CPU depth map with the root peaks): every frame is a
contiguous float32 [43, h, w] array, and +-inf or values whose centroid overflows appear only outside the root
planes, except in frames whose targets include "extract_only".  `connectable(hms, root_idx)` states the rule.
"""
import os
import sys

import numpy as np

H, W, NC, NJ, NL, MAXP = 128, 208, 43, 15, 14, 127
PAIRS = [0, 1, 0, 2, 0, 9, 9, 10, 10, 11, 0, 3, 3, 4, 4, 5, 2, 12, 12, 13, 13, 14, 2, 6, 6, 7, 7, 8]
BONE = np.array([26.42178982, 48.36980909, 14.88291009, 31.28002332, 23.915707, 14.97674918, 31.28002549, 23.91570732,
                 12.4644364, 48.26604433, 39.03553194, 12.4644364, 48.19076948, 39.03553252], np.float32)
F = np.float32
THR = F(0.2)


def near(h, w):
    """sqrtf(w * h) / 150 (bodyPartConnectorBase.cu:57)."""
    return F(np.sqrt(F(h * w))) / F(150)


NEAR = near(H, W)
NEAR_SCORE = F(0.1 + 1e-6)            # float(0.1f + 1e-6), :59
ROOTS = (0, 2)
EVEN = [j for j in range(NJ) if j % 2 == 0]
ODD = [j for j in range(NJ) if j % 2 == 1]


def up(v):
    return np.nextafter(F(v), F(np.inf))


def down(v):
    return np.nextafter(F(v), F(-np.inf))


def blank(h=H, w=W):
    return np.zeros((NC, h, w), np.float32)


def depth_map(seed, h=H, w=W):
    return np.random.default_rng(seed).uniform(0.5, 3, (h, w)).astype(np.float32)


def connectable(hms, root_idx):
    """The reference's connect reads rDepth[int(y)][int(x)] of every root peak: the root plane must be free of +-inf and
    of values large enough for the centroid sums to overflow.  NaN is safe (it is never a peak and never summed)."""
    p = hms[root_idx]
    fin = p[np.isfinite(p)]
    return not np.isinf(p).any() and (fin.size == 0 or float(np.abs(fin).max()) < 1e30)


# ---------------------------------------------------------------------------------------------------------------------
# float32 restatements used to place inputs (the tests measure with the oracle itself)
# ---------------------------------------------------------------------------------------------------------------------
def centroid(plane, y, x):
    """nmsBase.cu:93-126 for the peak at (y, x): 7x7 window clipped at the map, taps with score > 0, x*score + acc as
    one fused multiply-add (exact in float64 for the small windows this module builds, then rounded once)."""
    h, w = plane.shape
    xa = ya = sa = F(0)
    for yy in range(y - 3, y + 4):
        if 0 <= yy < h:
            for xx in range(x - 3, x + 4):
                if 0 <= xx < w and plane[yy, xx] > 0:
                    s = plane[yy, xx]
                    xa = F(xx * float(s) + float(xa))
                    ya = F(yy * float(s) + float(ya))
                    sa = F(sa + s)
    return F(F(xa / sa) + F(0.5)), F(F(ya / sa) + F(0.5))


def sample_count(a, b, h=H, w=W):
    """(n, norm, [(mX, mY, xs, ys)]) of the line integral from a = (x, y) to b (bodyPartConnectorBase.cu:16-37);
    xs, ys are the sample positions before the +0.5 and the truncation."""
    ax, ay = F(a[0]), F(a[1])
    dx, dy = F(F(b[0]) - ax), F(F(b[1]) - ay)
    dmax = max(abs(dx), abs(dy))
    n = int(F(np.sqrt(F(5) * dmax)) + F(0.5))
    n = max(5, min(25, n))
    norm = F(np.sqrt(F(float(dx) * float(dx) + float(F(dy * dy)))))
    sx, sy = F(dx / F(n)), F(dy / F(n))
    out = []
    for lm in range(n):
        xs, ys = F(lm * float(sx) + float(ax)), F(lm * float(sy) + float(ay))
        out.append((min(w - 1, int(F(xs + F(0.5)))), min(h - 1, int(F(ys + F(0.5)))), xs, ys))
    return n, norm, out


def _frame(name, hms, rd, *targets):
    return name, np.ascontiguousarray(hms, np.float32), np.ascontiguousarray(rd, np.float32), tuple(targets)


def _grid(step=4, lo=2, h=H, w=W):
    ys, xs = np.meshgrid(np.arange(lo, h - 1, step), np.arange(lo, w - 1, step), indexing="ij")
    return np.stack([ys.ravel(), xs.ravel()], 1)  # raster order


def _spread(default, n, lo=2, pitch=4):
    """Rows (or columns) for a layout drawn at 128 x 208: `default` where its last entry fits an axis of n pixels (an
    interior pixel with one more row below it), else as many as fit from `lo` on, `pitch` apart."""
    if max(default) <= n - 3:
        return list(default)
    return list(range(lo, n - 2, pitch))[:len(default)]


def _wrap(v, n):
    """v on an axis of n pixels, kept where its whole 7x7 window fits (3 ... n - 4); the identity where it already
    does."""
    return 3 + (v - 3) % (n - 6)


# Frames left out at a size, and why: (h, w, frame name) -> reason; filled in by the families as they are built.
LEFT_OUT = {}


def _leave_out(h, w, name, reason):
    LEFT_OUT[(h, w, name)] = reason


# ---------------------------------------------------------------------------------------------------------------------
# NMS
# ---------------------------------------------------------------------------------------------------------------------
def _cap_grid(h, w, need):
    """Single-pixel peak sites 4 px apart, or 2 px apart where that is too few for `need` (a zero between two sites is
    enough: every 3x3 neighbourhood holds one site)."""
    g = _grid(4, 2, h, w)
    return g if len(g) >= need else _grid(2, 2, h, w)


def nms_frames(h=H, w=W):
    rng = np.random.default_rng(11)
    # values at the threshold: isolated pixels at 0.2f - 1 ulp, 0.2f, 0.2f + 1 ulp (only the last is a peak)
    a = blank(h, w)
    vals = [down(THR), THR, up(THR)]
    pos = _grid(6, 3, h, w)[:90]
    for c in range(NJ):
        for i, (y, x) in enumerate(pos):
            a[c, y, x] = vals[(i + c) % 3]
    yield _frame("nms_threshold", a, depth_map(1, h, w), "nms.threshold")

    # plateaus: equal neighbours are never peaks (strict > against all eight); controls lift one pixel by one ulp.
    # Blocks sit in cells of 10 rows x 12 columns; a block whose cell does not fit the map is left out.
    shapes = {"h2": [(0, 0), (0, 1)], "v2": [(0, 0), (1, 0)], "d2": [(0, 0), (1, 1)], "a2": [(0, 1), (1, 0)],
              "row3": [(0, 0), (0, 1), (0, 2)], "l3": [(0, 0), (0, 1), (1, 0)], "sq4": [(0, 0), (0, 1), (1, 0), (1, 1)],
              "row4": [(0, 0), (0, 1), (0, 2), (0, 3)]}
    rows = min(12, (h - 6) // 10 + 1)
    a = blank(h, w)
    k = 0
    for c in range(NJ):
        for si, (nm, sh) in enumerate(shapes.items()):
            for vi, v in enumerate((F(0.5), F(0.15), up(THR), THR)):
                for ctrl in (0, 1):
                    y0, x0 = 4 + 10 * ((si * 2 + ctrl) % rows), 4 + 12 * (vi + 4 * ((si * 2 + ctrl) // rows)) + (c % 3)
                    if y0 + 1 <= h - 2 and x0 + 3 <= w - 2:
                        for dy, dx in sh:
                            a[c, y0 + dy, x0 + dx] = v
                        if ctrl:
                            dy, dx = sh[k % len(sh)]
                            a[c, y0 + dy, x0 + dx] = up(v)
                    k += 1
    yield _frame("nms_plateau", a, depth_map(2, h, w), "nms.plateau")

    # rows / columns 1 and h-2 / w-2 next to large border values (inside the 7x7 window, some inside the 3x3); on an
    # axis shorter than 32 pixels the peaks start at 2 instead of 6 and the border values sit two pixels before them;
    # on a large map they are spread further apart, so that the whole border fits under the 127-peak cap
    a = blank(h, w)
    step = 9
    while 2 * (len(range(6, w - 6, step)) + len(range(6, h - 6, step))) > 120:  # all of them under the 127 cap
        step += 1
    for c in range(NJ):
        for i, x in enumerate(range(6 + c % 4, w - 6, step) if w >= 32 else range(2 + c % 2, w - 3, step)):
            for y, yb in ((1, 0), (h - 2, h - 1)):
                a[c, y, x] = 0.6 + 0.01 * (i % 5)
                a[c, yb, x + (2 if i % 3 else 1)] = 5.0 + i  # i % 3 == 0: in the 3x3 neighbourhood, suppresses the peak
        for i, y in enumerate(range(6 + c % 4, h - 6, step) if h >= 32 else range(2 + c % 2, h - 3, step)):
            for x, xb in ((1, 0), (w - 2, w - 1)):
                a[c, y, x] = 0.55 + 0.01 * (i % 5)
                a[c, y + ((3 if i % 3 else -1) if h >= 32 else -2), xb] = 7.0 + i
        a[c, 0, 0] = a[c, 0, w - 1] = a[c, h - 1, 0] = a[c, h - 1, w - 1] = 9.0
    yield _frame("nms_border", a, depth_map(3, h, w), "nms.border")

    # centroid windows clipped by every edge and corner (distance 1, 2, 3 from the edge), windows full of small values
    a = blank(h, w)
    for c in range(NJ):
        d = 1 + c % 3
        pos = [(d, d), (d, w - 1 - d), (h - 1 - d, d), (h - 1 - d, w - 1 - d), (d, _wrap(60 + c, w)),
               (h - 1 - d, _wrap(90 + c, w)), (_wrap(40 + c, h), d), (_wrap(70 + c, h), w - 1 - d)]
        if min(h, w) < 16:  # the corner and edge windows would cover each other: corners in even planes only
            pos = pos[:4] if c % 2 == 0 else pos[4:]
        for y, x in pos:
            win = a[c, max(0, y - 3):y + 4, max(0, x - 3):x + 4]
            win[...] = rng.uniform(0.01, 0.19, win.shape)
            a[c, y, x] = 0.9
    yield _frame("nms_clipped", a, depth_map(4, h, w), "nms.clipped")

    # windows holding zeros, -0, negatives, NaN and denormals; +-inf and overflowing values outside the root planes
    mix = np.array([0.0, -0.0, -0.3, np.nan, 1e-40, 1e-45, 3e-39, 0.1, 0.15], np.float32)
    hot = np.array([np.inf, -np.inf, 3e38, np.nan, 1e-45], np.float32)
    sites = _grid(10, min(6, (min(h, w) - 1) // 2), h, w)[:150]  # windows on the last column or row are clipped

    def window_frame(hot_planes):
        a = blank(h, w)
        r = np.random.default_rng(12)
        for c in range(NJ):
            for i, (y, x) in enumerate(sites):
                win = a[c, y - 3:y + 4, x - 3:x + 4]
                win[...] = r.choice(mix, win.shape)
                if i % 7 == 3:  # a NaN neighbour suppresses the peak (every comparison with NaN is false)
                    win[2:5, 2:5] = r.choice(mix[:3], (3, 3))
                    win[2, 3] = np.nan
                else:
                    win[2:5, 2:5] = r.choice(np.delete(mix, 3), (3, 3))
                if c in hot_planes and i % 3 == 0 and win.shape == (7, 7):  # outside the 3x3: the peak survives,
                    # its centroid is inf or NaN
                    win[0, r.integers(0, 7)] = r.choice(hot)
                    win[6, 6] = r.choice(hot)
                a[c, y, x] = 0.8
        return a

    yield _frame("nms_window_values", window_frame([c for c in range(NJ) if c not in ROOTS]), depth_map(5, h, w),
                 "nms.window_values", "nms.nonfinite_centroid")
    yield _frame("nms_window_values_all_planes", window_frame(range(NJ)), depth_map(6, h, w), "nms.window_values",
                 "nms.nonfinite_centroid", "extract_only")

    # the 127-peak cap: 127, 128 and 300 peaks in one plane (as many as fit, at least 129), kept in raster order; 127
    # persons, 128 neck candidates
    g = _cap_grid(h, w, 300)
    if len(g) < 129:
        _leave_out(h, w, "nms_cap", "%d single-pixel peak sites fit, the cap needs 128 and one more" % len(g))
        _leave_out(h, w, "nms_saturated", "%d single-pixel peak sites fit, the cap needs 128" % len(g))
        return
    many = min(300, len(g))
    a = blank(h, w)
    for c, n in ((3, 127), (4, 128), (5, many), (2, 127), (0, 128), (12, many), (1, many)):
        sel = np.sort(rng.choice(len(g), n, replace=False))
        a[c, g[sel, 0], g[sel, 1]] = rng.uniform(0.3, 1.0, n)
    a[NJ::2] = 0.4
    a[NJ + 1::2] = 0.3
    yield _frame("nms_cap", a, depth_map(7, h, w), "nms.cap", "group.persons127")

    # every keypoint plane saturated (300 peaks each, or as many as fit), PAFs noise: all 14 limbs score 127 x 127 pairs
    a = blank(h, w)
    for c in range(NJ):
        sel = np.sort(rng.choice(len(g), many, replace=False))
        a[c, g[sel, 0], g[sel, 1]] = rng.uniform(0.3, 1.0, many)
    a[NJ:] = rng.normal(0.2, 0.5, (NC - NJ, h, w))
    yield _frame("nms_saturated", a, depth_map(8, h, w), "nms.saturated", "group.persons127")


# ---------------------------------------------------------------------------------------------------------------------
# PAF
# ---------------------------------------------------------------------------------------------------------------------
def _sym3(a, c, y, x):
    a[c, y - 1:y + 2, x - 1:x + 2] = [[0.1, 0.3, 0.1], [0.3, 0.9, 0.3], [0.1, 0.3, 0.1]]


def two_tap(p0, p1, u):
    """Centroid coordinate along one axis of a peak of value 1 at p0 with one more tap u at p1 > p0 on the same line
    (raster order: the peak is summed first): float(float(p1*u + p0) / float(1 + u)) + 0.5, vectorised over u."""
    u = np.asarray(u, np.float32)
    acc = (p1 * u.astype(np.float64) + p0).astype(np.float32)
    return ((acc / (np.float32(1) + u)).astype(np.float32) + np.float32(0.5)).astype(np.float32)


def straddle(p0, u_lo, u_hi, measure, limit, k=2):
    """Tap values for a B candidate at p0 with a tap at p0 + 3 whose measure(coordinate) lies just below `limit`
    (the k largest distinct values) and at or just above it (the k smallest)."""
    us = np.unique(np.linspace(u_lo, u_hi, 200001).astype(np.float32))
    m = measure(two_tap(p0, p0 + 3, us))
    vals, first = np.unique(m, return_index=True)
    below, above = first[vals < limit][-k:], first[vals >= limit][:k]
    return [us[i] for i in below] + [us[i] for i in above]


# sample counts: n = int(sqrtf(5 * d) + 0.5) reaches 25 from an offset d of 121 px on (24.5^2 / 5 = 120.05)
MAX_N_OFFSET = 121


def paf_frames(h=H, w=W):
    rng = np.random.default_rng(21)
    thr = near(h, w)
    # coincident candidates: the same single pixels and symmetric 3x3 windows in every keypoint plane (norm 0)
    a = blank(h, w)
    for c in range(NJ):
        for y, x in _grid(8, 4, h, w)[::3]:
            a[c, y, x] = 1.0
        for y, x in _grid(8, 8, h, w)[1::5]:
            _sym3(a, c, y, x)
    a[NJ:] = rng.normal(0.3, 0.3, (NC - NJ, h, w))
    yield _frame("paf_coincident", a, depth_map(21, h, w), "paf.coincident")

    # integer offsets along x, y and the diagonal: even planes at t = 0, 5, 10, 15 (every residue mod 4), odd planes at
    # t = 0, 4, 8, ...; the PAF points along the line, so forward pairs pass and backward ones fail.  The longest offset
    # is what the map holds: every sample count up to 25 needs one axis of at least MAX_N_OFFSET + 4 pixels.
    for nm, d, o, tmax in (("x", (0, 1), (min(20, h // 2), 2), min(200, w - 4)),
                           ("y", (1, 0), (2, min(20, w // 2)), min(124, h - 4)),
                           ("diag", (1, 1), (2, 2), min(124, min(h, w) - 4)),
                           ("anti", (-1, 1), (h - 3, 2), min(122, min(h, w) - 6))):
        a = blank(h, w)
        for c in range(NJ):
            ts = [0, 5, 10, 15] if c % 2 == 0 else range(0, tmax + 1, 4)
            for t in ts:
                if t <= tmax:
                    a[c, o[0] + d[0] * t, o[1] + d[1] * t] = 1.0
        nrm = np.hypot(*d)
        a[NJ::2] = d[1] / nrm * 0.7
        a[NJ + 1::2] = d[0] / nrm * 0.7
        yield _frame("paf_offsets_" + nm, a, depth_map(22, h, w), "paf.offsets")

    # direction sweeps: one A at the centre of even planes, B on circles in odd planes, a radial field (zero at A)
    a = blank(h, w)
    cy, cx = h // 2, w // 2
    pts = []
    for r in (12, 25, 40, 55):
        m = int(2 * np.pi * r / 4.6)
        for k in range(m):
            t = 2 * np.pi * k / m + 0.01 * r
            p = (int(round(cy + r * np.sin(t))), int(round(cx + r * np.cos(t))))
            inside = 1 <= p[0] < h - 1 and 1 <= p[1] < w - 1
            if inside and all(max(abs(p[0] - q[0]), abs(p[1] - q[1])) >= 4 for q in pts):
                pts.append(p)
    pts = np.array(pts)
    for c in range(NJ):
        if c % 2 == 0:
            a[c, cy, cx] = 1.0
        else:
            a[c, pts[:, 0], pts[:, 1]] = 1.0
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    ry, rx = yy - cy, xx - cx
    rr = np.hypot(ry, rx)
    rr[cy, cx] = np.inf
    a[NJ::2] = rx / rr * 0.9
    a[NJ + 1::2] = ry / rr * 0.9
    yield _frame("paf_angles", a, depth_map(23, h, w), "paf.angles")

    # rows along +x: projection == the PAF x value; 0.05f exactly and one ulp either side; 19 of 20 and 24 of 25.  On a
    # map with fewer rows the pairs move to rows 4 apart; a pair longer than the map is wide is left out.
    a = blank(h, w)
    spec = [(20, 10, 40, down(0.05)), (30, 10, 40, F(0.05)), (40, 10, 40, up(0.05)), (50, 10, 140, F(0.05)),
            (60, 10, 140, up(0.05)), (80, 10, 90, None), (90, 12, 92, None), (100, 10, 135, None),
            (110, 10, 135, None), (120, 10, 90, 0.8)]
    spec = [s for s in spec if s[2] <= w - 2]
    rows = {y: s[1:] for y, s in zip(_spread([s[0] for s in spec], h), spec)} if spec else {}
    for y, (xa, xb, v) in rows.items():
        for c in EVEN:
            a[c, y, xa] = 1.0
        for c in ODD:
            a[c, y, xb] = 1.0
        # the samples of a pair on row y read row y + 1 (centroids sit at pixel + 0.5, and the sampler adds 0.5)
        a[NJ::2, y + 1, :] = F(0.8) if v is None else F(v)
        if v is None:  # zero one sample of the pair: n - 1 of n samples pass
            n, _, smp = sample_count((xa + 0.5, y + 0.5), (xb + 0.5, y + 0.5), h, w)
            mx, my = smp[n // 2][:2]
            assert my == y + 1
            a[NJ::2, y + 1, mx] = 0
    if rows:
        yield _frame("paf_threshold_ratio", a, depth_map(24, h, w), "paf.threshold", "paf.ratio")
    else:
        _leave_out(h, w, "paf_threshold_ratio", "the shortest pair along x is 30 px long")

    # distances around the near threshold sqrtf(h*w)/150 and around the 1e-6 norm floor: A single pixels in even
    # planes, B a pixel k = floor(threshold) away plus a small tap 3 further that moves its centroid; the PAFs are zero.
    # Where the threshold is an integer (360 x 1000: exactly 4.0f) no tap is needed to reach it: paf_near_exact puts
    # single-pixel pairs exactly k - 1, k and k + 1 px apart along x and y (strict <: k scores -1, k - 1 the constant).
    a = blank(h, w)
    k = int(thr)
    frac = float(thr) - k
    xa0 = 20 if w >= 30 + k else 1  # column of A on the rows along x
    ya0 = 50 if h >= 60 + k else 1  # row of A on the columns along y
    xrows = _spread([10, 20, 30, 40], h)
    # on the right of the rows along x, clear of the norm-floor pairs at columns 1 ... 4
    ycols = [x for x in (60, 80, 100, 120) if x <= w - 2] or list(range(w - 3, xa0 + k + 8, -6))[:4]
    if frac > 0:
        # the bounds first chosen at 128 x 208; elsewhere around the tap value that puts B on the threshold
        u0 = frac / (3 - frac)
        lo, hi = (0.0298, 0.0305) if (h, w) == (H, W) else (u0 * 0.99, u0 * 1.01)
        u = straddle(xa0 + k, lo, hi, lambda b: np.float32(b - np.float32(xa0 + 0.5)), thr)
        if (h, w) != (H, W):  # a small map may hold fewer than four pairs: one on each side first, the axes opposite
            u = [u[i] for i in (0, 2, 1, 3)]
        for i, y in enumerate(xrows):  # along x: norm = |dx|
            for c in EVEN:
                a[c, y, xa0] = 1.0
            for c in ODD:
                a[c, y, xa0 + k] = 1.0
                a[c, y, xa0 + k + 3] = u[i]
        u = straddle(ya0 + k, lo, hi, lambda b: np.sqrt(np.float32(b - np.float32(ya0 + 0.5)) ** 2), thr)
        if (h, w) != (H, W):
            u = [u[i] for i in (2, 0, 3, 1)]
        for i, x0 in enumerate(ycols):  # along y: norm = sqrtf(dy * dy)
            for c in EVEN:
                a[c, ya0, x0] = 1.0
            for c in ODD:
                a[c, ya0 + k, x0] = 1.0
                a[c, ya0 + k + 3, x0] = u[i]
    else:
        for y, x0, dd in zip(xrows, ycols, (k - 1, k, k + 1)):
            for c in EVEN:
                a[c, y, xa0] = 1.0
                a[c, ya0, x0] = 1.0
            for c in ODD:
                a[c, y, xa0 + dd] = 1.0
                a[c, ya0 + dd, x0] = 1.0
    # norms of 7 ... 10 ulps of 1.5 (2^-23 each) straddle 1e-6: A at column 1, B on the same pixel with a tiny tap
    us = np.unique(np.linspace(1e-7, 6e-7, 20001).astype(np.float32))
    ulps = np.round((two_tap(1, 4, us) - np.float32(1.5)).astype(np.float64) * 2 ** 23).astype(int)
    for y, kk in zip(_spread([70, 80, 90, 100], h), (7, 8, 9, 10)):
        for c in EVEN:
            a[c, y, 1] = 1.0
        for c in ODD:
            a[c, y, 1] = 1.0
            a[c, y, 4] = us[np.flatnonzero(ulps == kk)[0]]
    if frac > 0:
        yield _frame("paf_near", a, depth_map(25, h, w), "paf.near", "paf.norm_floor")
    else:
        yield _frame("paf_near_exact", a, depth_map(25, h, w), "paf.near_exact", "paf.norm_floor")

    # NaN, +-inf and denormals in the PAF planes (never in the keypoint planes)
    g = _grid(4, 2, h, w)
    for i in range(2):
        r = np.random.default_rng(26 + i)
        a = blank(h, w)
        n = min(60, len(g))
        for c in range(NJ):
            sel = np.sort(r.choice(len(g), n, replace=False))
            a[c, g[sel, 0], g[sel, 1]] = r.uniform(0.3, 1.0, n)
        a[NJ:] = r.normal(0.3, 0.4, (NC - NJ, h, w))
        m = r.uniform(size=a[NJ:].shape)
        a[NJ:][m < 0.1] = np.nan
        a[NJ:][(m >= 0.1) & (m < 0.11)] = np.inf
        a[NJ:][(m >= 0.11) & (m < 0.12)] = -np.inf
        a[NJ:][(m >= 0.12) & (m < 0.13)] = 1e-40
        yield _frame("paf_nonfinite_%d" % i, a, depth_map(26 + i, h, w), "paf.nonfinite")


# ---------------------------------------------------------------------------------------------------------------------
# grouping
# ---------------------------------------------------------------------------------------------------------------------
def bone_dist(limb, depth):
    """association.cpp:198 in float64, stored as float."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return F(np.float64(1.2) * np.float64(BONE[limb]) / np.float64(F(depth)))


def exact_zero_depth(limb, limb_dist):
    """Root depth at which bone_dist / limb_dist / 4 - 1 == -0.5 exactly (a pair score of 0.5 then becomes 0)."""
    want = F(2 * limb_dist)
    d = F(1.2 * float(BONE[limb]) / float(want))
    for _ in range(64):
        b = bone_dist(limb, d)
        if b == want:
            return d
        d = up(d) if b > want else down(d)
    raise AssertionError("no float32 depth gives an exact zero score")


def root_sites(n, h, w):
    """n (y, x) pixels in raster order, spread over the map on a 4 px grid (each 7x7 centroid window sees one of them),
    or a 2 px grid where that is too few; None where fewer than n fit."""
    g = _cap_grid(h, w, n)
    if len(g) < n:
        return None
    return g[np.round(np.linspace(0, len(g) - 1, n)).astype(int)]


def sized_tie_frame(keys, root_ch, seed, h, w):
    """tests/test_assoc_limits_gpu.py:tie_frame at (h, w), the root peaks on root_sites: the root channel holds exactly
    len(keys) single-pixel peaks, peak i (raster order) on a root depth of keys[i]; the other keypoint channels are
    noise
    with many peaks, the PAFs point along +x.  None where the peaks do not fit."""
    pos = root_sites(len(keys), h, w)
    if pos is None:
        return None
    rng = np.random.default_rng(seed)
    lo = rng.normal(0, 1, (43, h // 4, w // 4)).astype(np.float32)
    hms = np.kron(lo, np.ones((1, 4, 4), np.float32)) * 0.4 + rng.normal(0, 0.15, (43, h, w)).astype(np.float32)
    hms[15::2] = 0.6 + 0.1 * hms[15::2]
    hms[16::2] *= 0.1
    hms[root_ch] = 0
    hms[root_ch, pos[:, 0], pos[:, 1]] = rng.uniform(0.5, 0.9, len(keys))
    rd = rng.uniform(0.5, 3, (h, w)).astype(np.float32)
    rd[pos[:, 0], pos[:, 1]] = keys
    return hms.astype(np.float32), rd


def group_frames(h=H, w=W):
    # a star of candidates on the +x and +y rays of the root (65 per plane, several per lane), PAFs 0.5 everywhere:
    # every ray candidate scores exactly 0.5, the first index must win.  Roots 0 and 2 coincide, so the limb between
    # them scores -1 and the chains hanging off the other root are cut.
    a = blank(h, w)
    y0, x0 = min(6, h - 2), 6
    for c in range(NJ):
        if c in ROOTS:
            a[c, y0, x0] = 1.0
        else:
            a[c, y0, x0 + 4 * np.arange(1, min(50, (w - 2 - x0) // 4 + 1))] = 1.0
            a[c, y0 + 4 * np.arange(1, min(30, (h - 2 - y0) // 4 + 1)), x0] = 1.0
    a[NJ:] = 0.5
    rd = depth_map(31, h, w)
    rd[y0, x0] = 1.0
    yield _frame("group_star", a, rd, "group.tie", "group.cut")

    # two persons competing for the same candidate: the one earlier in depth order takes it, the other gets the second
    # (equal scores as well, so without the `used` flag it would take the first again); both depth orders.  Two groups
    # of 13 rows each (persons on the first row, candidates 8 below, a PAF band over them) need 25 rows.
    if h < 25:
        _leave_out(h, w, "group_used_0", "two groups of persons and candidates need 25 rows")
        _leave_out(h, w, "group_used_1", "two groups of persons and candidates need 25 rows")
    ya, yb = (30, 90) if h >= 104 else (2, 15)
    xa = 40 if w >= 50 else 2
    for flip in (0, 1) if h >= 25 else ():
        a = blank(h, w)
        for c in range(NJ):
            if c in ROOTS:
                a[c, ya, xa] = a[c, ya, xa + 4] = 1.0
                a[c, yb, xa] = a[c, yb, xa + 4] = 1.0
            else:
                a[c, ya + 8, xa + 2] = a[c, ya + 8, xa + 6] = 1.0
                a[c, yb + 8, xa + 2] = a[c, yb + 8, xa + 6] = 1.0
        a[NJ + 1::2, ya - 2:ya + 11] = a[NJ + 1::2, yb - 2:yb + 11] = 0.5  # PAF bands: far pairs read zeros, score -1
        rd = depth_map(32 + flip, h, w)
        # shallow roots: bone_dist / limb_dist / 4 > 1, so the distance penalty is 0 and the scores stay equal
        rd[ya, xa], rd[ya, xa + 4] = (0.25, 0.3) if not flip else (0.3, 0.25)
        rd[yb, xa], rd[yb, xa + 4] = (0.35, 0.35)  # tied depths: the sort's order decides
        yield _frame("group_used_%d" % flip, a, rd, "group.used")

    # pair scores of 0.5 turned into exactly 0 and into the smallest positive value by the distance penalty
    # (limb_dist 8, bone_dist 16 and one ulp more); also a root at depth 0 (bone_dist inf)
    r1, r2 = (30, 80) if h >= 84 else (h // 3, 2 * h // 3)
    xr = 30 if w >= 40 else 2
    for k, nm in enumerate(("zero", "above", "depth0")):
        a = blank(h, w)
        rd = depth_map(34 + k, h, w)
        for root, dst, limb, y in ((2, 12, 8, r1), (0, 1, 0, r2)):
            a[root, y, xr] = 1.0
            a[dst, y, xr + 8] = 1.0
            d = exact_zero_depth(limb, 8.0)
            if k == 1:  # the largest depth whose bone_dist exceeds 16: the score is the smallest positive one
                while bone_dist(limb, d) == F(16):
                    d = down(d)
            rd[y, xr] = (d, d, 0.0)[k]
        a[NJ::2] = 0.5
        yield _frame("group_penalty_" + nm, a, rd, "group.zero_score")

    # the root-depth key sets of tests/golden/sort_cases.py (ties, +-0, NaN, +-inf, negatives, heap-sort fallback)
    import sort_cases

    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if here not in sys.path:
        sys.path.insert(0, here)
    from test_assoc_limits_gpu import tie_frame

    sets = sort_cases.key_sets()
    names = [nm for nm in sets if nm.endswith(("_n17", "_n127"))]
    for i, nm in enumerate(names):
        root = ROOTS[i % 2]
        fr = tie_frame(sets[nm], root, 700 + i) if (h, w) == (H, W) else sized_tie_frame(sets[nm], root, 700 + i, h, w)
        if fr is None:
            _leave_out(h, w, "group_keys_%s_root%d" % (nm, root), "%d root peaks 4 px apart do not fit" % len(sets[nm]))
            continue
        yield _frame("group_keys_%s_root%d" % (nm, root), fr[0], fr[1], "group.depth_keys")


# ---------------------------------------------------------------------------------------------------------------------
# breadth
# ---------------------------------------------------------------------------------------------------------------------
BREADTH_SEEDS = 32


def sized_random_heatmaps(seed, h, w):
    """tests/test_assoc_gpu.py:random_heatmaps (one frame) at (h, w): backbone-like noise, many peaks."""
    rng = np.random.default_rng(seed)
    lo = rng.normal(0, 1, (1, 43, h // 4, w // 4)).astype(np.float32)
    hms = np.kron(lo, np.ones((1, 1, 4, 4), np.float32)) * 0.4 + rng.normal(0, 0.15, (1, 43, h, w)).astype(np.float32)
    rd = rng.uniform(0.5, 3, (1, h, w)).astype(np.float32)
    return hms[0].astype(np.float32), rd[0]


def breadth_frames(h=H, w=W, seeds=BREADTH_SEEDS):
    """At 128 x 208 the frames of the other association tests; at other sizes the same generators at (h, w): the
    random_heatmaps and make_scene seeds, the crowded root channels where 150 root peaks fit, and the empty and
    saturated edge cases.  `seeds` trims the seeded frames (the first `seeds` of each)."""
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if here not in sys.path:
        sys.path.insert(0, here)
    from smap_b200.synth import make_scene

    if (h, w) == (H, W):
        from test_assoc_gpu import edge_cases, random_heatmaps
        from test_assoc_limits_gpu import crowded_frames

        for s in range(seeds):
            hms, rd = random_heatmaps(800 + s, B=1)
            yield _frame("random_%d" % s, hms[0], rd[0], "breadth")
        for s in range(seeds):
            sc = make_scene(900 + s, 15)
            yield _frame("scene_%d" % s, sc["hms"], sc["root_d"], "breadth")
        hms, rd = crowded_frames()
        for i in range(len(hms)):
            yield _frame("crowded_%d" % i, hms[i], rd[i], "breadth", "group.persons127")
        for nm, hms in edge_cases().items():
            yield _frame("edge_" + nm, hms, np.random.default_rng(3).uniform(0.5, 3, (H, W)).astype(np.float32),
                         "breadth")
        return
    import sort_cases

    for s in range(seeds):
        yield _frame("random_%d" % s, *sized_random_heatmaps(800 + s, h, w), "breadth")
    for s in range(seeds):
        sc = make_scene(900 + s, 15, h=h, w=w)
        yield _frame("scene_%d" % s, sc["hms"], sc["root_d"], "breadth")
    rng = np.random.default_rng(17)
    keys = [(0.5 + 0.25 * rng.permutation(np.arange(150) % 5)).astype(np.float32), sort_cases.heap_sort_keys(),
            sort_cases.key_sets()["few3_n127"]]
    for i, k in enumerate(keys):
        fr = sized_tie_frame(k, 2, 500 + i, h, w)
        if fr is None:
            _leave_out(h, w, "crowded_%d" % i, "%d root peaks 4 px apart do not fit" % len(k))
            continue
        yield _frame("crowded_%d" % i, fr[0], fr[1], "breadth", "group.persons127")
    rd = np.random.default_rng(3).uniform(0.5, 3, (h, w)).astype(np.float32)
    yield _frame("edge_empty", blank(h, w), rd, "breadth")
    b = blank(h, w)
    g = _grid(4, 2, h, w)
    for c in range(NJ):
        b[c, g[:, 0], g[:, 1]] = 0.5 + 0.001 * ((g[:, 1] + c) % 7)
    b[NJ:] = np.random.default_rng(0).normal(0, 0.5, (NC - NJ, h, w))
    yield _frame("edge_saturated_peaks", b, rd, "breadth")


FAMILIES = {"nms": nms_frames, "paf": paf_frames, "group": group_frames, "breadth": breadth_frames}


def frames(h=H, w=W, families=tuple(FAMILIES)):
    """Every frame of `families` at map size (h, w).  Frames that cannot reach their rule at this size are left out
    and recorded in LEFT_OUT[(h, w, name)] with the reason."""
    for f in families:
        yield from FAMILIES[f](h, w)
