"""The adversarial association frames (tests/golden/assoc_adversary.py) hold what they are built for, measured with the
oracle and by inspecting the inputs: a frame that no longer reaches its rule would let tests/test_assoc_reference_gpu.py
pass without checking that rule.  Also: where the reference sources exist, build() must have built the reference
extension, so that the GPU comparison cannot turn into skips."""
import os

import numpy as np
import pytest

import assoc_adversary as A
from oracle import assoc, build_ref

F = np.float32


@pytest.fixture(scope="module")
def fams():
    return {f: list(A.FAMILIES[f]()) for f in ("nms", "paf", "group")}


def by_name(fams, name):
    return next(fr for fam in fams.values() for fr in fam if fr[0] == name)


def peak_list(peaks, j):
    n = int(peaks[j, 0, 0])
    return peaks[j, 1:n + 1]


def pixels(peaks, j):
    """Peak pixels (y, x) of joint j, from centroids of isolated single pixels (x + 0.5, y + 0.5)."""
    p = peak_list(peaks, j)
    return [(int(y), int(x)) for x, y, _ in p]


def pair_scores(peaks, scores, l):
    a, b = A.PAIRS[2 * l], A.PAIRS[2 * l + 1]
    na, nb = int(peaks[a, 0, 0]), int(peaks[b, 0, 0])
    return peak_list(peaks, a), peak_list(peaks, b), scores[l, :na, :nb]


def test_reference_built_where_its_sources_exist():
    if not os.path.isdir(os.path.join(build_ref.REF, "extensions")):
        pytest.skip("no reference sources on this machine")
    assert build_ref.built_path() is not None, "build() did not build the reference extension (oracle/build_ref.py)"


def test_frames_are_safe_for_the_reference():
    names = set()
    for name, hms, rd, targets in A.frames():
        assert name not in names
        names.add(name)
        assert hms.shape == (43, A.H, A.W) and hms.dtype == np.float32 and hms.flags.c_contiguous, name
        assert rd.shape == (A.H, A.W) and rd.dtype == np.float32, name
        if "extract_only" not in targets:
            assert all(A.connectable(hms, r) for r in A.ROOTS), name
    assert 100 <= len(names) <= 300


def test_nms_threshold(fams):
    _, hms, _, _ = by_name(fams, "nms_threshold")
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        p = hms[c]
        assert (p == A.THR).sum() > 20 and (p == A.down(A.THR)).sum() > 20
        assert sorted(pixels(peaks, c)) == sorted(map(tuple, np.argwhere(p == A.up(A.THR))))


def test_nms_plateaus_give_no_peak(fams):
    _, hms, _, _ = by_name(fams, "nms_plateau")
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        p = hms[c]
        # a pixel is a peak iff it is the one-ulp control bump of a plateau above the threshold (the centroid of a
        # plateau's peak lies between its pixels, so peaks are matched by value)
        bumps = [tuple(q) for q in np.argwhere(p > A.THR)
                 if (p[q[0] - 1:q[0] + 2, q[1] - 1:q[1] + 2] == A.down(p[q[0], q[1]])).any()]
        assert len(bumps) == 24  # 8 shapes at 0.5, 0.2f + 1 ulp and 0.2f
        assert sorted(peak_list(peaks, c)[:, 2]) == sorted(p[q] for q in bumps)
        flat = [q for q in np.argwhere(p > A.THR) if tuple(q) not in bumps]
        assert len(flat) > 40 and (p[tuple(np.array(flat).T)] <= 0.5).all()


def test_nms_border(fams):
    _, hms, _, _ = by_name(fams, "nms_border")
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        ys = [int(y) for _, y, _ in peak_list(peaks, c)]
        xs = [int(x) for x, _, _ in peak_list(peaks, c)]
        p = hms[c]
        border_max = max(p[0].max(), p[-1].max(), p[:, 0].max(), p[:, -1].max())
        assert border_max > peak_list(peaks, c)[:, 2].max()  # the largest values never become peaks
        # a pixel next to a larger border pixel in its 3x3 is no peak; the others are, pulled toward the border
        inner = [tuple(q) for q in np.argwhere(p > A.THR) if 0 < q[0] < A.H - 1 and 0 < q[1] < A.W - 1]
        free = [q for q in inner if p[q] > np.delete(p[q[0] - 1:q[0] + 2, q[1] - 1:q[1] + 2].ravel(), 4).max()]
        assert sorted(peak_list(peaks, c)[:, 2]) == sorted(p[q] for q in free) and 10 < len(free) < len(inner)
        assert min(ys) < 1.5 and max(ys) > A.H - 2.5 and min(xs) < 1.5 and max(xs) > A.W - 2.5
        assert len(peak_list(peaks, c)) < int((p[1:-1, 1:-1] > A.THR).sum())


def test_nms_windows_clipped_by_every_edge_and_corner(fams):
    _, hms, _, _ = by_name(fams, "nms_clipped")
    seen = set()
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        for x, y, _ in peak_list(peaks, c):
            px, py = int(x), int(y)
            seen.add(((py < 3) - (py > A.H - 4), (px < 3) - (px > A.W - 4)))
    assert {(a, b) for a in (-1, 0, 1) for b in (-1, 0, 1)} - {(0, 0)} <= seen


def test_nms_window_values(fams):
    _, hms, _, _ = by_name(fams, "nms_window_values")
    peaks, _ = assoc.extract(hms)
    kinds = set()
    for c in range(A.NJ):
        for y, x in np.argwhere(hms[c] == F(0.8)):
            win = hms[c, y - 3:y + 4, x - 3:x + 4]
            kinds |= {k for k, m in (("zero", win == 0), ("negzero", (win == 0) & np.signbit(win)), ("neg", win < 0),
                                     ("nan", np.isnan(win)), ("denormal", (win != 0) & (np.abs(win) < 1.2e-38)))
                      if m.any()}
        co = peak_list(peaks, c)[:, :2]
        if c in A.ROOTS:
            assert np.isfinite(co).all()
        else:
            assert np.isinf(co).any() and np.isnan(co).any(), c
    assert kinds == {"zero", "negzero", "neg", "nan", "denormal"}
    # a NaN among the eight neighbours suppresses the peak
    assert int(peaks[0, 0, 0]) < int((hms[0] == F(0.8)).sum())


def test_nms_cap_keeps_raster_order(fams):
    _, hms, _, _ = by_name(fams, "nms_cap")
    peaks, _ = assoc.extract(hms)
    for c, n in ((3, 127), (4, 128), (5, 300), (2, 127), (0, 128)):
        px = [tuple(q) for q in np.argwhere(hms[c] > A.THR)]  # argwhere is raster order
        assert len(px) == n and int(peaks[c, 0, 0]) == 127
        assert pixels(peaks, c) == px[:127]
        if n > 127:
            assert px[127] not in pixels(peaks, c)  # the 128th raster peak exists and is dropped
    assert len(assoc.connect(hms, by_name(fams, "nms_cap")[2], 2)) == 127


def test_nms_saturated(fams):
    _, hms, rd, _ = by_name(fams, "nms_saturated")
    peaks, scores = assoc.extract(hms)
    assert all(int(peaks[c, 0, 0]) == 127 for c in range(A.NJ))
    assert all((pair_scores(peaks, scores, l)[2] > 0).any() for l in range(A.NL))


def test_paf_coincident(fams):
    _, hms, _, _ = by_name(fams, "paf_coincident")
    peaks, scores = assoc.extract(hms)
    n = 0
    for l in range(A.NL):
        pa, pb, s = pair_scores(peaks, scores, l)
        same = (pa[:, None, 0] == pb[None, :, 0]) & (pa[:, None, 1] == pb[None, :, 1])
        assert (s[same] == -1).all()
        n += int(same.sum())
    assert n > 14 * 50
    # the symmetric 3x3 windows put their centroids off the pixel grid
    assert any(float(x) % 1 != 0.5 for x, _, _ in peak_list(peaks, 0))


def test_paf_offsets_reach_every_sample_count(fams):
    ns, ds, trans = set(), set(), set()
    for name in ("paf_offsets_x", "paf_offsets_y", "paf_offsets_diag", "paf_offsets_anti"):
        _, hms, _, _ = by_name(fams, name)
        peaks, scores = assoc.extract(hms)
        pa, pb, s = pair_scores(peaks, scores, 0)
        for a in pa:
            for b in pb:
                n, norm, _ = A.sample_count(a[:2], b[:2])
                d = float(max(abs(b[0] - a[0]), abs(b[1] - a[1])))
                ns.add(n)
                ds.add(d)
                trans.add((d, n))
        assert (s > 0.5).any() and (s == -1).any()
    assert ns == set(range(5, 26))
    assert set(range(0, 141)) <= ds
    # both sides of every change of n
    for n in range(5, 25):
        assert any(m == n for _, m in trans) and any(m == n + 1 for _, m in trans)


def test_paf_angles_land_on_half_pixels(fams):
    _, hms, _, _ = by_name(fams, "paf_angles")
    peaks, scores = assoc.extract(hms)
    pa, pb, s = pair_scores(peaks, scores, 0)
    half = 0
    counts = set()
    for a in pa:
        for b in pb:
            n, _, smp = A.sample_count(a[:2], b[:2])
            half += sum(1 for _, _, xs, ys in smp if float(xs) % 1 == 0.5 or float(ys) % 1 == 0.5)
    assert half > 50
    assert len(pb) > 60 and (s > 0).sum() > 10 and (s == -1).sum() > 10


def test_paf_threshold_and_ratio(fams):
    _, hms, _, _ = by_name(fams, "paf_threshold_ratio")
    peaks, scores = assoc.extract(hms)
    pa, pb, s = pair_scores(peaks, scores, 0)

    def score(y, xa, xb):
        i = [k for k, p in enumerate(pa) if p[1] == y + 0.5 and p[0] == xa + 0.5][0]
        j = [k for k, p in enumerate(pb) if p[1] == y + 0.5 and p[0] == xb + 0.5][0]
        return s[i, j]

    assert hms[15, 31, 20] == F(0.05) and score(30, 10, 40) == -1 and score(50, 10, 140) == -1
    assert score(40, 10, 40) > 0.05 and score(60, 10, 140) > 0  # (25 samples of 0.05f + 1 ulp average to below it)
    assert score(20, 10, 40) == -1
    # 19 of 20: ratio exactly 0.95f, refused; 24 of 25 accepted; 20 of 20 accepted
    for y, xa, xb, want_n, want_c in ((80, 10, 90, 20, 19), (90, 12, 92, 20, 19), (100, 10, 135, 25, 24),
                                      (110, 10, 135, 25, 24)):
        n, _, smp = A.sample_count((xa + 0.5, y + 0.5), (xb + 0.5, y + 0.5))
        c = sum(1 for mx, my, _, _ in smp if hms[15, my, mx] > F(0.05))
        assert (n, c) == (want_n, want_c)
        if n == 20:
            assert F(c) / F(n) == F(0.95) and score(y, xa, xb) == -1
        else:
            assert abs(score(y, xa, xb) - F(0.8)) < 1e-6
    assert abs(score(120, 10, 90) - F(0.8)) < 1e-6


def test_paf_near_threshold(fams):
    _, hms, _, _ = by_name(fams, "paf_near")
    peaks, scores = assoc.extract(hms)
    pa, pb, s = pair_scores(peaks, scores, 0)
    near_below, near_above, floor = [], [], {}
    for i, a in enumerate(pa):
        for j, b in enumerate(pb):
            _, norm, _ = A.sample_count(a[:2], b[:2])
            if abs(float(norm) - float(A.NEAR)) < 1e-3:
                (near_below if norm < A.NEAR else near_above).append((float(A.NEAR - norm), s[i, j]))
            if 0 < norm < 2e-6:
                floor[float(norm)] = s[i, j]
    assert len(near_below) >= 4 and len(near_above) >= 4
    assert all(v == A.NEAR_SCORE for _, v in near_below) and all(v == -1 for _, v in near_above)
    assert min(d for d, _ in near_below) < 3e-6 and max(d for d, _ in near_above) > -3e-6  # one step either side
    assert any(d == 0 for d, _ in near_above) or max(d for d, _ in near_above) > -3e-6
    # norms straddling the 1e-6 floor: refused at or below it, the near constant above it
    assert sorted(floor.items()) == [(k * 2.0 ** -23, -1 if k * 2.0 ** -23 <= 1e-6 else A.NEAR_SCORE) for k in (7, 8, 9, 10)]


def test_paf_nonfinite(fams):
    for name in ("paf_nonfinite_0", "paf_nonfinite_1"):
        _, hms, _, _ = by_name(fams, name)
        assert np.isnan(hms[15:]).any() and np.isinf(hms[15:]).any() and np.isfinite(hms[:15]).all()
        peaks, scores = assoc.extract(hms)
        s = np.concatenate([pair_scores(peaks, scores, l)[2].ravel() for l in range(A.NL)])
        assert (s > 0).sum() > 20 and np.isinf(s).any()


def test_group_ties_first_index_wins(fams):
    _, hms, rd, _ = by_name(fams, "group_star")
    peaks, scores = assoc.extract(hms)
    for root, limb, dst in ((2, 8, 12), (0, 0, 1)):
        _, pb, s = pair_scores(peaks, scores, limb)
        row = s[0]
        assert (row == 0.5).sum() == len(pb) > 64  # every candidate ties, in every lane and across lanes
        for flag in (False, True):
            b = assoc.connect(hms, rd, root, flag)
            assert len(b) == 1
            assert tuple(b[0, dst, :2]) == tuple(pb[0, :2])  # the first index
        # chains through the other root are cut: it coincides with this root, so it scores -1 and is never joined
        other = 2 - root
        b = assoc.connect(hms, rd, root, True)
        assert b[0, other, 3] == 0
        cut = [12, 6] if root == 0 else [1, 9, 3]
        assert (b[0, cut, 3] == 0).all()


def test_group_used_flags_decide(fams):
    for flip in (0, 1):
        _, hms, rd, _ = by_name(fams, "group_used_%d" % flip)
        peaks, scores = assoc.extract(hms)
        _, pb, s = pair_scores(peaks, scores, 8)
        b = assoc.connect(hms, rd, 2, True)
        first = [p for p in range(len(b)) if b[p, 2, 1] == 30.5][0]
        second = [p for p in range(len(b)) if b[p, 2, 1] == 30.5][1]
        assert first < second and b[first, 2, 0] == (40.5 if not flip else 44.5)
        assert b[first, 12, 0] == 42.5 and b[second, 12, 0] == 46.5  # the second person's best is taken
        ridx = [k for k, p in enumerate(peak_list(peaks, 2)) if p[0] == b[second, 2, 0] and p[1] == 30.5][0]
        c1 = [k for k, p in enumerate(pb) if p[0] == 42.5 and p[1] == 38.5][0]
        assert s[ridx, c1] == s[ridx].max() > 0


def test_group_penalty_reaches_exact_zero(fams):
    res = {}
    for nm in ("zero", "above", "depth0"):
        _, hms, rd, _ = by_name(fams, "group_penalty_" + nm)
        for root, dst, limb, y in ((2, 12, 8, 30), (0, 1, 0, 80)):
            bd = A.bone_dist(limb, rd[y, 30])
            with np.errstate(divide="ignore"):
                t = F(F(F(bd / F(8)) / F(4)) - F(1))
            b = assoc.connect(hms, rd, root, True)
            res[nm, root] = (float(F(0.5) + min(t, F(0))), float(b[0, dst, 3]))
            assert assoc.connect(hms, rd, root, False)[0, dst, 3] == 1
    for root in (0, 2):
        assert res["zero", root] == (0.0, 0.0)  # score exactly 0: refused (strict > 0)
        assert 0 < res["above", root][0] < 1e-6 and res["above", root][1] == 1
        assert res["depth0", root] == (0.5, 1.0)  # bone_dist inf: no penalty


def test_group_depth_keys_and_capacity(fams):
    import sort_cases

    frames = [f for f in fams["group"] if "group.depth_keys" in f[3]]
    kinds = {f[0].split("_")[2] for f in frames}
    assert {"equal", "few3", "nan1", "nans", "pm0", "infneg", "heap"} <= kinds
    assert {int(f[0][-1]) for f in frames} == {0, 2}
    for name, hms, rd, _ in frames[::4]:
        root = int(name[-1])
        keys = rd[hms[root] > A.THR]
        assert sort_cases.has_tie(keys), name
    name, hms, rd, _ = by_name(fams, "group_keys_heap_n127_root0")
    assert len(assoc.connect(hms, rd, 0)) == 127
