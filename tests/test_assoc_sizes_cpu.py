"""The adversarial association frames at map sizes other than 128x208 (tests/golden/assoc_adversary.py, frames(h, w))
hold what they are built for, measured with the oracle and by inspecting the inputs; the 128x208 frames are still the
ones tests/test_assoc_reference_gpu.py was written against; and the reference module that runs at other sizes
(dapalib_ref_dims, oracle/build_ref.py) was built and accepts exactly the sizes at which the reference is
deterministic.  tests/test_assoc_sizes_gpu.py runs the kernels, the oracle and that module on these frames."""
import hashlib
import os

import numpy as np
import pytest

import assoc_adversary as A
from oracle import assoc, build_ref
from test_assoc_adversary_cpu import pair_scores, peak_list, pixels
from test_assoc_sizes_gpu import SIZES

F = np.float32
OTHER = [(h, w) for h, w, _, _ in SIZES if (h, w) != (A.H, A.W)]
IDS = ["%dx%d" % s for s in OTHER]

# sha256 over the sha256 of each frame's name, heat maps, depth map and targets, in order: taken from frames() at
# 128x208 before the module took a size
DIGEST_128x208 = "742af76c5508d23dfc8f55729c6b2a65976af6fb4823328351ce46bb87060c2d"

# frames left out per size; every other frame is built at every size
LEFT_OUT = {
    (8, 64): {"nms_cap", "nms_saturated", "group_used_0", "group_used_1", "crowded_0", "crowded_1", "crowded_2"} |
             {"group_keys_%s_n127_root%d" % (k, r) for k, r in (("equal", 2), ("few2", 0), ("few3", 2), ("few4", 0),
                                                                 ("few5", 2), ("nan1", 0), ("nans", 2), ("pm0", 0),
                                                                 ("infneg", 2), ("heap", 0))},
    (256, 16): {"paf_threshold_ratio"},
    (32, 32): {"paf_threshold_ratio"},
}


def digest(frames):
    hs = hashlib.sha256()
    n = 0
    for name, hms, rd, targets in frames:
        for x in (name.encode(), hms.tobytes(), rd.tobytes(), repr(targets).encode()):
            hs.update(hashlib.sha256(x).digest())
        n += 1
    return n, hs.hexdigest()


_cache = {}


def fams(h, w):
    if (h, w) not in _cache:
        _cache.clear()  # one size at a time: 360 x 1000 frames take 62 MB each
        _cache[(h, w)] = {f: {fr[0]: fr for fr in A.FAMILIES[f](h, w)} for f in ("nms", "paf", "group")}
    return _cache[(h, w)]


def frame(h, w, name):
    fs = fams(h, w)
    return next(fam[name] for fam in fs.values() if name in fam)


# ---------------------------------------------------------------------------------------------------------------------
def test_frames_at_128x208_are_unchanged():
    assert digest(A.frames()) == (114, DIGEST_128x208)
    assert digest(A.frames(A.H, A.W)) == (114, DIGEST_128x208)


def test_dims_module_built_where_the_reference_sources_exist():
    if not os.path.isdir(os.path.join(build_ref.REF, "extensions")):
        pytest.skip("no reference sources on this machine")
    assert build_ref.dims_built_path() is not None, "build() did not build dapalib_ref_dims (oracle/build_ref.py)"
    assert build_ref.built_path() != build_ref.dims_built_path()


def test_setter_accepts_exactly_the_deterministic_sizes():
    """w % 16 == 0 (no racing border writes in nmsRegisterKernel) and h*w % 512 == 0 (no partial block in
    writeResultKernel, whose __syncthreads() sits inside `if (globalIdx < length)`), on every multiple of 8 up to 1024
    and on the sizes of the GPU file.  A refused size leaves the module's size as it was.  No GPU is needed."""
    r = build_ref.load_ref_dims()
    if r is None:
        pytest.skip("dapalib_ref_dims is not built here (no reference sources)")
    _, set_size = r
    try:
        for h, w, live, _ in SIZES:
            assert (set_size(h, w) == 0) == live, (h, w)
        assert set_size(A.H, A.W) == 0
        cur = (A.H, A.W)
        for h in range(8, 1025, 8):
            for w in range(8, 1025, 8):
                want = 2 if w % 16 else 3 if (h * w) % 512 else 0
                got = set_size(h, w)
                assert got == want, (h, w, got)
                cur = (h, w) if want == 0 else cur
                assert set_size.get() == cur
        assert set_size(128, 208) == 0
        for h, w in ((2, 512), (512, 2), (0, 0), (-16, 32)):
            assert set_size(h, w) == 1 and set_size.get() == (128, 208)
    finally:
        set_size(A.H, A.W)
    assert set_size.get() == (A.H, A.W)


@pytest.mark.parametrize("h,w", OTHER, ids=IDS)
def test_frames_are_safe_for_the_reference(h, w):
    names = set()
    for name, hms, rd, targets in A.frames(h, w, families=("nms", "paf", "group")):
        assert name not in names
        names.add(name)
        assert hms.shape == (43, h, w) and hms.dtype == np.float32 and hms.flags.c_contiguous, name
        assert rd.shape == (h, w) and rd.dtype == np.float32 and rd.flags.c_contiguous, name
        if "extract_only" not in targets:
            assert all(A.connectable(hms, r) for r in A.ROOTS), name
    for name, hms, rd, targets in A.breadth_frames(h, w, seeds=1):
        assert hms.shape == (43, h, w) and rd.shape == (h, w) and all(A.connectable(hms, r) for r in A.ROOTS), name
    left = {k[2] for k in A.LEFT_OUT if k[:2] == (h, w)}
    assert left == LEFT_OUT.get((h, w), set())
    assert all(A.LEFT_OUT[(h, w, n)] for n in left)  # every one with its reason


# ---------------------------------------------------------------------------------------------------------------------
# NMS
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", OTHER, ids=IDS)
def test_nms_rules(h, w):
    _, hms, _, _ = frame(h, w, "nms_threshold")
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        p = hms[c]
        assert (p == A.THR).any() and (p == A.down(A.THR)).any()
        assert sorted(pixels(peaks, c)) == sorted(map(tuple, np.argwhere(p == A.up(A.THR))))

    _, hms, _, _ = frame(h, w, "nms_plateau")
    peaks, _ = assoc.extract(hms)
    for c in range(A.NJ):
        p = hms[c]
        bumps = [tuple(q) for q in np.argwhere(p > A.THR)
                 if (p[max(0, q[0] - 1):q[0] + 2, max(0, q[1] - 1):q[1] + 2] == A.down(p[q[0], q[1]])).any()]
        assert bumps and sorted(peak_list(peaks, c)[:, 2]) == sorted(p[q] for q in bumps)
        assert any(tuple(q) not in bumps for q in np.argwhere(p > A.THR))  # a plateau pixel that is no peak

    _, hms, _, _ = frame(h, w, "nms_border")
    peaks, _ = assoc.extract(hms)
    edges = set()
    for c in range(A.NJ):
        p = hms[c]
        inner = [tuple(q) for q in np.argwhere(p > A.THR) if 0 < q[0] < h - 1 and 0 < q[1] < w - 1]
        free = [q for q in inner if p[q] > np.delete(p[q[0] - 1:q[0] + 2, q[1] - 1:q[1] + 2].ravel(), 4).max()]
        assert list(peak_list(peaks, c)[:, 2]) == [p[q] for q in free][:127] and 0 < len(free) < len(inner)
        assert len(free) <= 127  # the whole border is under the cap
        for x, y, _ in peak_list(peaks, c):
            edges |= {e for e, hit in (("top", y < 1.5), ("bottom", y > h - 2.5), ("left", x < 1.5),
                                        ("right", x > w - 2.5)) if hit}
    assert edges == {"top", "bottom", "left", "right"}

    _, hms, _, _ = frame(h, w, "nms_clipped")
    peaks, _ = assoc.extract(hms)
    seen = set()
    for c in range(A.NJ):
        for x, y, _ in peak_list(peaks, c):
            px, py = int(x), int(y)
            seen.add(((py < 3) - (py > h - 4), (px < 3) - (px > w - 4)))
    assert {(a, b) for a in (-1, 0, 1) for b in (-1, 0, 1)} - {(0, 0)} <= seen

    _, hms, _, _ = frame(h, w, "nms_window_values")
    peaks, _ = assoc.extract(hms)
    kinds, nonfinite = set(), set()
    for c in range(A.NJ):
        for y, x in np.argwhere(hms[c] == F(0.8)):
            win = hms[c, max(0, y - 3):y + 4, max(0, x - 3):x + 4]
            kinds |= {k for k, m in (("zero", win == 0), ("negzero", (win == 0) & np.signbit(win)), ("neg", win < 0),
                                     ("nan", np.isnan(win)), ("denormal", (win != 0) & (np.abs(win) < 1.2e-38)))
                      if m.any()}
        co = peak_list(peaks, c)[:, :2]
        if c in A.ROOTS:
            assert np.isfinite(co).all()
        else:
            nonfinite |= {k for k, m in (("inf", np.isinf(co)), ("nan", np.isnan(co))) if m.any()}
    assert kinds == {"zero", "negzero", "neg", "nan", "denormal"} and nonfinite == {"inf", "nan"}

    if (h, w) in LEFT_OUT and "nms_cap" in LEFT_OUT[(h, w)]:
        return
    _, hms, rd, _ = frame(h, w, "nms_cap")
    peaks, _ = assoc.extract(hms)
    for c, n in ((3, 127), (4, 128), (2, 127), (0, 128), (5, None)):
        px = [tuple(q) for q in np.argwhere(hms[c] > A.THR)]  # raster order
        assert (n is None and len(px) > 128) or len(px) == n
        # raster order, matched by value: on a 2 px grid the neighbours pull the centroids off their pixels
        assert int(peaks[c, 0, 0]) == 127 and list(peak_list(peaks, c)[:, 2]) == [hms[c][q] for q in px[:127]]
    assert len(assoc.connect(hms, rd, 2)) == 127
    _, hms, _, _ = frame(h, w, "nms_saturated")
    peaks, scores = assoc.extract(hms)
    assert all(int(peaks[c, 0, 0]) == 127 for c in range(A.NJ))
    assert all((pair_scores(peaks, scores, l)[2] > 0).any() for l in range(A.NL))


# ---------------------------------------------------------------------------------------------------------------------
# PAF
# ---------------------------------------------------------------------------------------------------------------------
def expected_row_score(hms, a, b, h, w):
    """The score of a pair on one row (dy = 0, so the projection is the x plane's value), restated in float32 from the
    inputs: count the samples above 0.05f, accept above a 0.95 ratio with their float32 mean, else the near constant
    below the threshold, else -1."""
    n, norm, smp = A.sample_count(a, b, h, w)
    vals = [hms[15, my, mx] for mx, my, _, _ in smp if hms[15, my, mx] > F(0.05)]
    if F(len(vals)) / F(n) > F(0.95):
        s = F(0)
        for v in vals:
            s = F(s + v)
        return F(s / F(len(vals)))
    return A.NEAR_SCORE if norm < A.near(h, w) else F(-1)


@pytest.mark.parametrize("h,w", OTHER, ids=IDS)
def test_paf_rules(h, w):
    _, hms, _, _ = frame(h, w, "paf_coincident")
    peaks, scores = assoc.extract(hms)
    n = 0
    for l in range(A.NL):
        pa, pb, s = pair_scores(peaks, scores, l)
        same = (pa[:, None, 0] == pb[None, :, 0]) & (pa[:, None, 1] == pb[None, :, 1])
        assert (s[same] == -1).all()
        n += int(same.sum())
    assert n >= 14

    # offsets: every sample count from 5 up to the count of the longest offset the map holds (25 from 121 px on)
    ns, longest = set(), 0
    for name in ("paf_offsets_x", "paf_offsets_y", "paf_offsets_diag", "paf_offsets_anti"):
        _, hms, _, _ = frame(h, w, name)
        peaks, scores = assoc.extract(hms)
        pa, pb, s = pair_scores(peaks, scores, 0)
        for a in pa:
            for b in pb:
                ns.add(A.sample_count(a[:2], b[:2], h, w)[0])
                longest = max(longest, float(max(abs(b[0] - a[0]), abs(b[1] - a[1]))))
        assert (s == -1).any()
    top = max(5, min(25, int(np.sqrt(5 * longest) + 0.5)))
    assert ns == set(range(5, top + 1))
    assert (top == 25) == (max(h, w) - 4 >= A.MAX_N_OFFSET)

    _, hms, _, _ = frame(h, w, "paf_angles")
    peaks, scores = assoc.extract(hms)
    pa, pb, s = pair_scores(peaks, scores, 0)
    half = sum(1 for a in pa for b in pb for _, _, xs, ys in A.sample_count(a[:2], b[:2], h, w)[2]
               if float(xs) % 1 == 0.5 or float(ys) % 1 == 0.5)
    assert half > 0 and len(pb) > 0 and (s == -1).any()

    if "paf_threshold_ratio" not in LEFT_OUT.get((h, w), ()):
        _, hms, _, _ = frame(h, w, "paf_threshold_ratio")
        peaks, scores = assoc.extract(hms)
        pa, pb, s = pair_scores(peaks, scores, 0)
        seen = 0
        for i, a in enumerate(pa):
            for j, b in enumerate(pb):
                if a[1] == b[1]:
                    assert s[i, j] == expected_row_score(hms, a[:2], b[:2], h, w), (a, b)
                    seen += 1
        assert seen >= 1

    near = A.near(h, w)
    if float(near) == int(near):
        # exact equality on the pixel lattice: pairs k - 1, k, k + 1 px apart along x and y
        _, hms, _, _ = frame(h, w, "paf_near_exact")
        peaks, scores = assoc.extract(hms)
        pa, pb, s = pair_scores(peaks, scores, 0)
        got = {}
        for i, a in enumerate(pa):
            for j, b in enumerate(pb):
                _, norm, _ = A.sample_count(a[:2], b[:2], h, w)
                axis = "x" if a[1] == b[1] else "y" if a[0] == b[0] else None
                if axis and abs(float(norm) - float(near)) <= 1:
                    got[(axis, float(norm))] = s[i, j]
        k = float(near)
        assert got == {(ax, d): (A.NEAR_SCORE if d < k else F(-1)) for ax in "xy" for d in (k - 1, k, k + 1)}
    else:
        _, hms, _, _ = frame(h, w, "paf_near")
        peaks, scores = assoc.extract(hms)
        pa, pb, s = pair_scores(peaks, scores, 0)
        below, above = [], []
        for i, a in enumerate(pa):
            for j, b in enumerate(pb):
                _, norm, _ = A.sample_count(a[:2], b[:2], h, w)
                if abs(float(norm) - float(near)) < 1e-3 and norm > 1e-5:
                    (below if norm < near else above).append((float(near - norm), s[i, j]))
        assert len(below) >= 1 and len(above) >= 1
        assert all(v == A.NEAR_SCORE for _, v in below) and all(v == -1 for _, v in above)
        step = 3e-6 * max(1.0, float(near))  # one float step either side
        assert min(d for d, _ in below) < step and max(d for d, _ in above) > -step
    # norms straddling the 1e-6 floor
    floor = {}
    for i, a in enumerate(pa):
        for j, b in enumerate(pb):
            _, norm, _ = A.sample_count(a[:2], b[:2], h, w)
            if 0 < norm < 2e-6:
                floor[float(norm)] = s[i, j]
    assert floor and all(v == (-1 if k <= 1e-6 else A.NEAR_SCORE) for k, v in floor.items())
    assert min(floor) <= 1e-6 < max(floor) or (len(floor) == 1 and h < 16)  # 8x64: one row holds one pair

    for name in ("paf_nonfinite_0", "paf_nonfinite_1"):
        _, hms, _, _ = frame(h, w, name)
        peaks, scores = assoc.extract(hms)
        s = np.concatenate([pair_scores(peaks, scores, l)[2].ravel() for l in range(A.NL)])
        assert (s > 0).any() and np.isnan(hms[15:]).any() and np.isinf(hms[15:]).any()


# ---------------------------------------------------------------------------------------------------------------------
# grouping
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", OTHER, ids=IDS)
def test_group_rules(h, w):
    _, hms, rd, _ = frame(h, w, "group_star")
    peaks, scores = assoc.extract(hms)
    for root, limb, dst in ((2, 8, 12), (0, 0, 1)):
        _, pb, s = pair_scores(peaks, scores, limb)
        assert (s[0] == 0.5).sum() == len(pb) > 1
        for flag in (False, True):
            b = assoc.connect(hms, rd, root, flag)
            assert len(b) == 1 and tuple(b[0, dst, :2]) == tuple(pb[0, :2])  # the first index
        assert assoc.connect(hms, rd, root, True)[0, 2 - root, 3] == 0

    if "group_used_0" not in LEFT_OUT.get((h, w), ()):
        ya, xa = (30 if h >= 104 else 2) + 0.5, (40 if w >= 50 else 2) + 0.5  # the layout assoc_adversary draws
        for flip in (0, 1):
            _, hms, rd, _ = frame(h, w, "group_used_%d" % flip)
            b = assoc.connect(hms, rd, 2, True)
            rows = [p for p in range(len(b)) if b[p, 2, 1] == ya]
            first, second = rows[0], rows[1]
            assert b[first, 2, 0] == (xa if not flip else xa + 4)
            assert b[first, 12, 0] == xa + 2 and b[second, 12, 0] == xa + 6  # the second person's best is taken

    res = {}
    r1, r2 = (30, 80) if h >= 84 else (h // 3, 2 * h // 3)
    xr = 30 if w >= 40 else 2
    for nm in ("zero", "above", "depth0"):
        _, hms, rd, _ = frame(h, w, "group_penalty_" + nm)
        for root, dst, limb, y in ((2, 12, 8, r1), (0, 1, 0, r2)):
            bd = A.bone_dist(limb, rd[y, xr])
            with np.errstate(divide="ignore"):
                t = F(F(F(bd / F(8)) / F(4)) - F(1))
            b = assoc.connect(hms, rd, root, True)
            res[nm, root] = (float(F(0.5) + min(t, F(0))), float(b[0, dst, 3]))
            assert assoc.connect(hms, rd, root, False)[0, dst, 3] == 1
    for root in (0, 2):
        assert res["zero", root] == (0.0, 0.0)
        assert 0 < res["above", root][0] < 1e-6 and res["above", root][1] == 1
        assert res["depth0", root] == (0.5, 1.0)

    import sort_cases

    keys = [f for f in fams(h, w)["group"].values() if "group.depth_keys" in f[3]]
    assert {int(f[0][-1]) for f in keys} == {0, 2}
    for name, hms, rd, _ in keys:
        root = int(name[-1])
        assert sort_cases.has_tie(rd[hms[root] > A.THR]), name
    if "group_keys_heap_n127_root0" in fams(h, w)["group"]:
        _, hms, rd, _ = frame(h, w, "group_keys_heap_n127_root0")
        assert len(assoc.connect(hms, rd, 0)) == 127


def test_near_threshold_is_exactly_4_at_360x1000():
    """sqrtf(360 * 1000) / 150 == 4.0f: the one size of the GPU file where `<` and `<=` differ on the pixel lattice."""
    assert A.near(360, 1000) == F(4) and float(A.near(128, 208)) != int(A.near(128, 208))
    assert "paf_near_exact" in {f[0] for f in A.paf_frames(360, 1000)}
