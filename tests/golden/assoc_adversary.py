"""Adversarial association frames: [43, 128, 208] float32 heat maps with [128, 208] root-depth maps, built so that each
rule of the reference association (extensions/gpu/nmsBase.cu, gpu/bodyPartConnectorBase.cu, association.cpp) is reached
where a restatement could misread it.  Seeded and deterministic; numpy only, apart from the breadth family, which reuses
the frames the other association tests build.

Every frame is (name, hms, rdepth, targets); `targets` names the rules the frame is built to reach.  tests/
test_assoc_adversary_cpu.py checks with the oracle that each family reaches them; tests/test_assoc_reference_gpu.py
runs the kernels, the oracle and the live reference extension on them.

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
contiguous float32 [43, 128, 208] array, and +-inf or values whose centroid overflows appear only outside the root
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
NEAR = F(np.sqrt(F(H * W))) / F(150)  # bodyPartConnectorBase.cu:57 at 128 x 208
NEAR_SCORE = F(0.1 + 1e-6)            # float(0.1f + 1e-6), :59
ROOTS = (0, 2)
EVEN = [j for j in range(NJ) if j % 2 == 0]
ODD = [j for j in range(NJ) if j % 2 == 1]


def up(v):
    return np.nextafter(F(v), F(np.inf))


def down(v):
    return np.nextafter(F(v), F(-np.inf))


def blank():
    return np.zeros((NC, H, W), np.float32)


def depth_map(seed):
    return np.random.default_rng(seed).uniform(0.5, 3, (H, W)).astype(np.float32)


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
    xa = ya = sa = F(0)
    for yy in range(y - 3, y + 4):
        if 0 <= yy < H:
            for xx in range(x - 3, x + 4):
                if 0 <= xx < W and plane[yy, xx] > 0:
                    s = plane[yy, xx]
                    xa = F(xx * float(s) + float(xa))
                    ya = F(yy * float(s) + float(ya))
                    sa = F(sa + s)
    return F(F(xa / sa) + F(0.5)), F(F(ya / sa) + F(0.5))


def sample_count(a, b):
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
        out.append((min(W - 1, int(F(xs + F(0.5)))), min(H - 1, int(F(ys + F(0.5)))), xs, ys))
    return n, norm, out


def _frame(name, hms, rd, *targets):
    return name, np.ascontiguousarray(hms, np.float32), np.ascontiguousarray(rd, np.float32), tuple(targets)


def _grid(step=4, lo=2):
    ys, xs = np.meshgrid(np.arange(lo, H - 1, step), np.arange(lo, W - 1, step), indexing="ij")
    return np.stack([ys.ravel(), xs.ravel()], 1)  # raster order


# ---------------------------------------------------------------------------------------------------------------------
# NMS
# ---------------------------------------------------------------------------------------------------------------------
def nms_frames():
    rng = np.random.default_rng(11)
    # values at the threshold: isolated pixels at 0.2f - 1 ulp, 0.2f, 0.2f + 1 ulp (only the last is a peak)
    a = blank()
    vals = [down(THR), THR, up(THR)]
    pos = _grid(6, 3)[:90]
    for c in range(NJ):
        for i, (y, x) in enumerate(pos):
            a[c, y, x] = vals[(i + c) % 3]
    yield _frame("nms_threshold", a, depth_map(1), "nms.threshold")

    # plateaus: equal neighbours are never peaks (strict > against all eight); controls lift one pixel by one ulp
    shapes = {"h2": [(0, 0), (0, 1)], "v2": [(0, 0), (1, 0)], "d2": [(0, 0), (1, 1)], "a2": [(0, 1), (1, 0)],
              "row3": [(0, 0), (0, 1), (0, 2)], "l3": [(0, 0), (0, 1), (1, 0)], "sq4": [(0, 0), (0, 1), (1, 0), (1, 1)],
              "row4": [(0, 0), (0, 1), (0, 2), (0, 3)]}
    a = blank()
    k = 0
    for c in range(NJ):
        for si, (nm, sh) in enumerate(shapes.items()):
            for vi, v in enumerate((F(0.5), F(0.15), up(THR), THR)):
                for ctrl in (0, 1):
                    y0, x0 = 4 + 10 * ((si * 2 + ctrl) % 12), 4 + 12 * (vi + 4 * ((si * 2 + ctrl) // 12)) + (c % 3)
                    for dy, dx in sh:
                        a[c, y0 + dy, x0 + dx] = v
                    if ctrl:
                        dy, dx = sh[k % len(sh)]
                        a[c, y0 + dy, x0 + dx] = up(v)
                    k += 1
    yield _frame("nms_plateau", a, depth_map(2), "nms.plateau")

    # rows / columns 1 and h-2 / w-2 next to large border values (inside the 7x7 window, some inside the 3x3)
    a = blank()
    for c in range(NJ):
        for i, x in enumerate(range(6 + c % 4, W - 6, 9)):
            for y, yb in ((1, 0), (H - 2, H - 1)):
                a[c, y, x] = 0.6 + 0.01 * (i % 5)
                a[c, yb, x + (2 if i % 3 else 1)] = 5.0 + i  # i % 3 == 0: in the 3x3 neighbourhood, suppresses the peak
        for i, y in enumerate(range(6 + c % 4, H - 6, 9)):
            for x, xb in ((1, 0), (W - 2, W - 1)):
                a[c, y, x] = 0.55 + 0.01 * (i % 5)
                a[c, y + (3 if i % 3 else -1), xb] = 7.0 + i
        a[c, 0, 0] = a[c, 0, W - 1] = a[c, H - 1, 0] = a[c, H - 1, W - 1] = 9.0
    yield _frame("nms_border", a, depth_map(3), "nms.border")

    # centroid windows clipped by every edge and corner (distance 1, 2, 3 from the edge), windows full of small values
    a = blank()
    for c in range(NJ):
        d = 1 + c % 3
        for y, x in [(d, d), (d, W - 1 - d), (H - 1 - d, d), (H - 1 - d, W - 1 - d), (d, 60 + c), (H - 1 - d, 90 + c),
                     (40 + c, d), (70 + c, W - 1 - d)]:
            win = a[c, max(0, y - 3):y + 4, max(0, x - 3):x + 4]
            win[...] = rng.uniform(0.01, 0.19, win.shape)
            a[c, y, x] = 0.9
    yield _frame("nms_clipped", a, depth_map(4), "nms.clipped")

    # windows holding zeros, -0, negatives, NaN and denormals; +-inf and overflowing values outside the root planes
    mix = np.array([0.0, -0.0, -0.3, np.nan, 1e-40, 1e-45, 3e-39, 0.1, 0.15], np.float32)
    hot = np.array([np.inf, -np.inf, 3e38, np.nan, 1e-45], np.float32)

    def window_frame(hot_planes):
        a = blank()
        r = np.random.default_rng(12)
        for c in range(NJ):
            for i, (y, x) in enumerate(_grid(10, 6)[:150]):
                win = a[c, y - 3:y + 4, x - 3:x + 4]
                win[...] = r.choice(mix, win.shape)
                if i % 7 == 3:  # a NaN neighbour suppresses the peak (every comparison with NaN is false)
                    win[2:5, 2:5] = r.choice(mix[:3], (3, 3))
                    win[2, 3] = np.nan
                else:
                    win[2:5, 2:5] = r.choice(np.delete(mix, 3), (3, 3))
                if c in hot_planes and i % 3 == 0:  # outside the 3x3: the peak survives, its centroid is inf or NaN
                    win[0, r.integers(0, 7)] = r.choice(hot)
                    win[6, 6] = r.choice(hot)
                a[c, y, x] = 0.8
        return a

    yield _frame("nms_window_values", window_frame([c for c in range(NJ) if c not in ROOTS]), depth_map(5),
                 "nms.window_values", "nms.nonfinite_centroid")
    yield _frame("nms_window_values_all_planes", window_frame(range(NJ)), depth_map(6), "nms.window_values",
                 "nms.nonfinite_centroid", "extract_only")

    # the 127-peak cap: 127, 128 and 300 peaks in one plane, kept in raster order; 127 persons, 128 neck candidates
    a = blank()
    g = _grid(4, 2)
    for c, n in ((3, 127), (4, 128), (5, 300), (2, 127), (0, 128), (12, 300), (1, 300)):
        sel = np.sort(rng.choice(len(g), n, replace=False))
        a[c, g[sel, 0], g[sel, 1]] = rng.uniform(0.3, 1.0, n)
    a[NJ::2] = 0.4
    a[NJ + 1::2] = 0.3
    yield _frame("nms_cap", a, depth_map(7), "nms.cap", "group.persons127")

    # every keypoint plane saturated (300 peaks each), PAFs noise: all 14 limbs score 127 x 127 pairs
    a = blank()
    for c in range(NJ):
        sel = np.sort(rng.choice(len(g), 300, replace=False))
        a[c, g[sel, 0], g[sel, 1]] = rng.uniform(0.3, 1.0, 300)
    a[NJ:] = rng.normal(0.2, 0.5, (NC - NJ, H, W))
    yield _frame("nms_saturated", a, depth_map(8), "nms.saturated", "group.persons127")


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


def paf_frames():
    rng = np.random.default_rng(21)
    # coincident candidates: the same single pixels and symmetric 3x3 windows in every keypoint plane (norm 0)
    a = blank()
    for c in range(NJ):
        for y, x in _grid(8, 4)[::3]:
            a[c, y, x] = 1.0
        for y, x in _grid(8, 8)[1::5]:
            _sym3(a, c, y, x)
    a[NJ:] = rng.normal(0.3, 0.3, (NC - NJ, H, W))
    yield _frame("paf_coincident", a, depth_map(21), "paf.coincident")

    # integer offsets along x, y and the diagonal: even planes at t = 0, 5, 10, 15 (every residue mod 4), odd planes at
    # t = 0, 4, 8, ...; the PAF points along the line, so forward pairs pass and backward ones fail
    for nm, d, o, tmax in (("x", (0, 1), (20, 2), 200), ("y", (1, 0), (2, 20), 124), ("diag", (1, 1), (2, 2), 124),
                           ("anti", (-1, 1), (125, 2), 122)):
        a = blank()
        for c in range(NJ):
            ts = [0, 5, 10, 15] if c % 2 == 0 else range(0, tmax + 1, 4)
            for t in ts:
                a[c, o[0] + d[0] * t, o[1] + d[1] * t] = 1.0
        nrm = np.hypot(*d)
        a[NJ::2] = d[1] / nrm * 0.7
        a[NJ + 1::2] = d[0] / nrm * 0.7
        yield _frame("paf_offsets_" + nm, a, depth_map(22), "paf.offsets")

    # direction sweeps: one A at the centre of even planes, B on circles in odd planes, a radial field (zero at A)
    a = blank()
    cy, cx = 64, 104
    pts = []
    for r in (12, 25, 40, 55):
        m = int(2 * np.pi * r / 4.6)
        for k in range(m):
            t = 2 * np.pi * k / m + 0.01 * r
            p = (int(round(cy + r * np.sin(t))), int(round(cx + r * np.cos(t))))
            if 1 <= p[0] < H - 1 and all(max(abs(p[0] - q[0]), abs(p[1] - q[1])) >= 4 for q in pts):
                pts.append(p)
    pts = np.array(pts)
    for c in range(NJ):
        if c % 2 == 0:
            a[c, cy, cx] = 1.0
        else:
            a[c, pts[:, 0], pts[:, 1]] = 1.0
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    ry, rx = yy - cy, xx - cx
    rr = np.hypot(ry, rx)
    rr[cy, cx] = np.inf
    a[NJ::2] = rx / rr * 0.9
    a[NJ + 1::2] = ry / rr * 0.9
    yield _frame("paf_angles", a, depth_map(23), "paf.angles")

    # rows along +x: projection == the PAF x value; 0.05f exactly and one ulp either side; 19 of 20 and 24 of 25
    a = blank()
    rows = {20: (10, 40, down(0.05)), 30: (10, 40, F(0.05)), 40: (10, 40, up(0.05)), 50: (10, 140, F(0.05)),
            60: (10, 140, up(0.05)), 80: (10, 90, None), 90: (12, 92, None), 100: (10, 135, None), 110: (10, 135, None),
            120: (10, 90, 0.8)}
    for y, (xa, xb, v) in rows.items():
        for c in EVEN:
            a[c, y, xa] = 1.0
        for c in ODD:
            a[c, y, xb] = 1.0
        # the samples of a pair on row y read row y + 1 (centroids sit at pixel + 0.5, and the sampler adds 0.5)
        a[NJ::2, y + 1, :] = F(0.8) if v is None else F(v)
        if v is None:  # zero one sample of the pair: n - 1 of n samples pass
            n, _, smp = sample_count((xa + 0.5, y + 0.5), (xb + 0.5, y + 0.5))
            mx, my = smp[n // 2][:2]
            assert my == y + 1
            a[NJ::2, y + 1, mx] = 0
    yield _frame("paf_threshold_ratio", a, depth_map(24), "paf.threshold", "paf.ratio")

    # distances around the near threshold sqrtf(128*208)/150 and around the 1e-6 norm floor: A single pixels in even
    # planes, B a pixel 1 away plus a small tap 3 further that moves its centroid; the PAFs are zero
    a = blank()
    x0, u = 20, straddle(21, 0.0298, 0.0305, lambda b: np.float32(b - np.float32(20.5)), NEAR)
    for i, y in enumerate((10, 20, 30, 40)):  # along x: norm = |dx|
        for c in EVEN:
            a[c, y, x0] = 1.0
        for c in ODD:
            a[c, y, x0 + 1] = 1.0
            a[c, y, x0 + 4] = u[i]
    y0 = 50  # along y: norm = sqrtf(dy * dy)
    u = straddle(y0 + 1, 0.0298, 0.0305, lambda b: np.sqrt(np.float32(b - np.float32(y0 + 0.5)) ** 2), NEAR)
    for i, x0 in enumerate((60, 80, 100, 120)):
        for c in EVEN:
            a[c, y0, x0] = 1.0
        for c in ODD:
            a[c, y0 + 1, x0] = 1.0
            a[c, y0 + 4, x0] = u[i]
    # norms of 7 ... 10 ulps of 1.5 (2^-23 each) straddle 1e-6: A at column 1, B on the same pixel with a tiny tap
    us = np.unique(np.linspace(1e-7, 6e-7, 20001).astype(np.float32))
    ulps = np.round((two_tap(1, 4, us) - np.float32(1.5)).astype(np.float64) * 2 ** 23).astype(int)
    for i, k in enumerate((7, 8, 9, 10)):
        y = 70 + 10 * i
        for c in EVEN:
            a[c, y, 1] = 1.0
        for c in ODD:
            a[c, y, 1] = 1.0
            a[c, y, 4] = us[np.flatnonzero(ulps == k)[0]]
    yield _frame("paf_near", a, depth_map(25), "paf.near", "paf.norm_floor")

    # NaN, +-inf and denormals in the PAF planes (never in the keypoint planes)
    for i in range(2):
        r = np.random.default_rng(26 + i)
        a = blank()
        for c in range(NJ):
            sel = np.sort(r.choice(len(_grid()), 60, replace=False))
            a[c, _grid()[sel, 0], _grid()[sel, 1]] = r.uniform(0.3, 1.0, 60)
        a[NJ:] = r.normal(0.3, 0.4, (NC - NJ, H, W))
        m = r.uniform(size=a[NJ:].shape)
        a[NJ:][m < 0.1] = np.nan
        a[NJ:][(m >= 0.1) & (m < 0.11)] = np.inf
        a[NJ:][(m >= 0.11) & (m < 0.12)] = -np.inf
        a[NJ:][(m >= 0.12) & (m < 0.13)] = 1e-40
        yield _frame("paf_nonfinite_%d" % i, a, depth_map(26 + i), "paf.nonfinite")


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


def group_frames():
    # a star of candidates on the +x and +y rays of the root (65 per plane, several per lane), PAFs 0.5 everywhere:
    # every ray candidate scores exactly 0.5, the first index must win.  Roots 0 and 2 coincide, so the limb between
    # them scores -1 and the chains hanging off the other root are cut.
    a = blank()
    y0, x0 = 6, 6
    for c in range(NJ):
        if c in ROOTS:
            a[c, y0, x0] = 1.0
        else:
            a[c, y0, x0 + 4 * np.arange(1, 50)] = 1.0
            a[c, y0 + 4 * np.arange(1, 30), x0] = 1.0
    a[NJ:] = 0.5
    rd = depth_map(31)
    rd[y0, x0] = 1.0
    yield _frame("group_star", a, rd, "group.tie", "group.cut")

    # two persons competing for the same candidate: the one earlier in depth order takes it, the other gets the second
    # (equal scores as well, so without the `used` flag it would take the first again); both depth orders
    for flip in (0, 1):
        a = blank()
        for c in range(NJ):
            if c in ROOTS:
                a[c, 30, 40] = a[c, 30, 44] = 1.0
                a[c, 90, 40] = a[c, 90, 44] = 1.0
            else:
                a[c, 38, 42] = a[c, 38, 46] = 1.0
                a[c, 98, 42] = a[c, 98, 46] = 1.0
        a[NJ + 1::2, 28:41] = a[NJ + 1::2, 88:101] = 0.5  # PAF bands: the far pairs read zeros and score -1
        rd = depth_map(32 + flip)
        # shallow roots: bone_dist / limb_dist / 4 > 1, so the distance penalty is 0 and the scores stay equal
        rd[30, 40], rd[30, 44] = (0.25, 0.3) if not flip else (0.3, 0.25)
        rd[90, 40], rd[90, 44] = (0.35, 0.35)  # tied depths: the sort's order decides
        yield _frame("group_used_%d" % flip, a, rd, "group.used")

    # pair scores of 0.5 turned into exactly 0 and into the smallest positive value by the distance penalty
    # (limb_dist 8, bone_dist 16 and one ulp more); also a root at depth 0 (bone_dist inf)
    for k, nm in enumerate(("zero", "above", "depth0")):
        a = blank()
        rd = depth_map(34 + k)
        for root, dst, limb, y in ((2, 12, 8, 30), (0, 1, 0, 80)):
            a[root, y, 30] = 1.0
            a[dst, y, 38] = 1.0
            d = exact_zero_depth(limb, 8.0)
            if k == 1:  # the largest depth whose bone_dist exceeds 16: the score is the smallest positive one
                while bone_dist(limb, d) == F(16):
                    d = down(d)
            rd[y, 30] = (d, d, 0.0)[k]
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
        hms, rd = tie_frame(sets[nm], root, 700 + i)
        yield _frame("group_keys_%s_root%d" % (nm, root), hms, rd, "group.depth_keys")


# ---------------------------------------------------------------------------------------------------------------------
# breadth
# ---------------------------------------------------------------------------------------------------------------------
def breadth_frames():
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if here not in sys.path:
        sys.path.insert(0, here)
    from smap_b200.synth import make_scene
    from test_assoc_gpu import edge_cases, random_heatmaps
    from test_assoc_limits_gpu import crowded_frames

    for s in range(32):
        hms, rd = random_heatmaps(800 + s, B=1)
        yield _frame("random_%d" % s, hms[0], rd[0], "breadth")
    for s in range(32):
        sc = make_scene(900 + s, 15)
        yield _frame("scene_%d" % s, sc["hms"], sc["root_d"], "breadth")
    hms, rd = crowded_frames()
    for i in range(len(hms)):
        yield _frame("crowded_%d" % i, hms[i], rd[i], "breadth", "group.persons127")
    for nm, hms in edge_cases().items():
        yield _frame("edge_" + nm, hms, np.random.default_rng(3).uniform(0.5, 3, (H, W)).astype(np.float32), "breadth")


FAMILIES = {"nms": nms_frames, "paf": paf_frames, "group": group_frames, "breadth": breadth_frames}


def frames(families=tuple(FAMILIES)):
    for f in families:
        yield from FAMILIES[f]()
