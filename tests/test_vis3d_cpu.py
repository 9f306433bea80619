"""CPU: the 3D panel oracle (oracle/view3d_numpy.py) on hand-built records, the composite against cv2.imencode, and
run_inference --vis_3d's host logic (argument parsing, frames too wide for the composite)."""
import os

import numpy as np
import pytest

from oracle import jpeg_encode_numpy as E
from oracle import render_numpy as R
from oracle import view3d_numpy as V
from smap_b200 import run_inference as ri

RECORD_DTYPE = np.dtype([("pred3d", "<f8", (127, 15, 4)), ("root_depth", "<f8", (127,)), ("pred2d", "<f4", (127, 15, 4)),
                         ("count", "<i4"), ("pad_", "<i4")])
RED, GREEN = R.PALETTE[0], R.PALETTE[1]


def record(persons):
    """persons: list of {joint: (X, Y, Z)} (score 1)."""
    r = np.zeros((), RECORD_DTYPE)
    r["count"] = len(persons)
    for p, joints in enumerate(persons):
        for j, xyz in joints.items():
            r["pred3d"][p, j] = tuple(xyz) + (1,)
    return r


def non_white(img):
    return ~(img == 255).all(-1)


def test_x_runs_across_and_z_goes_up():
    # P = 200: m = 10, avail = 179, r = 1.  Neck (0) to head (1) along +X: a run on the middle row from x = 10 to 189
    out = V.panel(record([{0: (0, 0, 0), 1: (1, 0, 0)}]), 200)
    ys, xs = np.nonzero(non_white(out))
    assert set(ys) == {99, 100, 101} and xs.min() == 9 and xs.max() == 190
    assert (out[100, 10:190] == RED).all()
    # the same limb along +Z: one column, the head (larger Z) nearer the top
    (a, b, colour), = V.elements(record([{0: (0, 0, 0), 1: (0, 0, 1)}]), 200)[12:]
    assert a[0] == b[0] == 100 and (a[1], b[1]) == (189, 10) and colour == RED
    # +Y goes down the panel (screen up is Z - Y)
    (a, b, _), = V.elements(record([{0: (0, 0, 0), 1: (0, 1, 0)}]), 200)[12:]
    assert a[0] == b[0] and a[1] < b[1]


def crossing(shift0, shift1):
    """Person 0's limb along X and person 1's along Z - Y cross at the panel point of (0, 0, 0) plus their shifts along
    (0, 1, 1), which moves a limb away from the viewer without moving it on the panel."""
    s0, s1 = np.array([0, 1, 1.0]) * shift0, np.array([0, 1, 1.0]) * shift1
    rec = record([{0: (-1, 0, 0) + s0, 1: (1, 0, 0) + s0}, {0: (0, 0.5, -0.5) + s1, 1: (0, -0.5, 0.5) + s1}])
    project, _ = V.fit(rec, 200)
    x, y = project(0, 0, 0)
    assert project(*(np.array([0, 0, 0.0]) + s1)) == (x, y)
    return V.panel(rec, 200), x, y


def test_nearer_limbs_cover_farther_ones_and_ties_go_in_row_order():
    out, x, y = crossing(0, 3)  # person 1 farther: under person 0
    assert (out[y, x] == RED).all() and (out[y - 20, x] == GREEN).all()
    out, x, y = crossing(3, 0)  # person 0 farther: under person 1
    assert (out[y, x] == GREEN).all() and (out[y, x - 20] == RED).all()
    out, x, y = crossing(0, 0)  # as far: row order, person 1 last
    assert (out[y, x] == GREEN).all()
    # within one person, equal depths paint in limb order: limbs 0 (0-1) and 1 (0-2), both at depth 0
    rec = record([{0: (0, 0, 0), 1: (1, 0, 0), 2: (-1, 0, 0)}])
    assert [e[2] for e in V.elements(rec, 200)] == [V.GREY] * 12 + [RED, RED]
    assert V.drawn_limbs(rec) == [(0, 0), (0, 1)]


def test_unplaced_joints_and_their_limbs_are_skipped():
    good = {0: (0, 0, 0), 1: (1, 0, 0), 2: (0, 1, 0)}
    clean = record([good])
    bad = record([{**good, 9: (5, 5, 5), 3: (np.nan, 0, 0), 12: (0, np.inf, 0), 6: (0, 0, 2e15)}])
    bad["pred3d"][0, 9, 3] = 0  # score 0: left out as gen_3d_pose's zeroed joints are
    assert V.drawn_limbs(bad) == V.drawn_limbs(clean) == [(0, 0), (0, 1)]
    assert (V.panel(bad, 300) == V.panel(clean, 300)).all()
    edge = record([{**good, 9: (0, 0, 1e15)}])  # |.| <= 1e15 is placed
    assert (0, 2) in V.drawn_limbs(edge)


def test_no_drawn_limb_gives_a_white_panel():
    white = np.full((120, 120, 3), 255, np.uint8)
    assert (V.panel(record([]), 120) == white).all()
    assert (V.panel(record([{0: (0, 0, 0), 5: (1, 1, 1)}]), 120) == white).all(), "joints without a limb"
    r = record([{0: (0, 0, 0), 1: (1, 0, 0)}])
    r["count"] = 0
    assert (V.panel(r, 120) == white).all(), "rows past count are not drawn"
    assert V.fit(r, 120) is None


def test_a_zero_length_limb_lands_at_the_centre():
    out = V.panel(record([{0: (3, 4, 5), 1: (3, 4, 5)}]), 201)  # span 0: k = 0, centre m + avail / 2 = 100
    ys, xs = np.nonzero(non_white(out))
    assert sorted(zip(ys, xs)) == [(99, 100), (100, 99), (100, 100), (100, 101), (101, 100)]
    assert (out[ys, xs] == RED).all()


def test_box_corners_sit_at_the_fit_extremes():
    rng = np.random.default_rng(4)
    rec = record([{j: (rng.uniform(-1, 1), 0, rng.uniform(0, 3)) for j in range(15)}])  # Y = 0: the box is a rectangle
    P = 400
    project, box = V.fit(rec, P)
    pts = [project(*rec["pred3d"][0, j, :3]) for j in range(15)]
    xs, ys = [p[0] for p in pts], [p[1] for p in pts]
    corners = {c for edge in box for c in edge}
    assert corners == {(x, y) for x in (min(xs), max(xs)) for y in (min(ys), max(ys))}
    m, avail = P // 20, P - 1 - 2 * (P // 20)
    assert (min(ys), max(ys)) == (m, m + avail), "the taller extent fills the panel"
    assert abs((min(xs) + max(xs)) - (P - 1)) <= 1, "the other one is centred"
    r = max(1, P // 400)
    ys_, xs_ = np.nonzero(non_white(V.panel(rec, P)))
    assert (xs_.min(), xs_.max(), ys_.min(), ys_.max()) == (min(xs) - r, max(xs) + r, min(ys) - r, max(ys) + r)
    # with depth spread too, the box's projection reaches past the joints' own extent
    rec["pred3d"][0, :, 1] = rng.uniform(-1, 1, 15)
    _, box = V.fit(rec, P)
    assert len(box) == 12


@pytest.mark.parametrize("P", [1, 2, 3])
def test_tiny_panels(P):
    rec = record([{0: (0, 0, 0), 1: (1, 2, 3), 2: (-1, 5, 0)}])
    f = np.zeros((P, 5, 3), np.uint8)
    out = V.render_view3d(f, rec, row(5, P))
    assert out.shape == (P, 5 + P, 3)
    assert non_white(out[:, 5:]).any()


def row(w, h, nw=832, nh=512):
    s = min(nw / w, nh / h)
    return np.array([s, w, h, nw, nh, w, w, w / 2, h / 2])


def random_record(rng, n, w, h, nw=832, nh=512):
    r = np.zeros((), RECORD_DTYPE)
    r["count"] = n
    r["pred2d"][:n, :, 0] = rng.uniform(0, nw, (n, 15))
    r["pred2d"][:n, :, 1] = rng.uniform(0, nh, (n, 15))
    r["pred2d"][:n, :, 3] = rng.random((n, 15)) < 0.9
    r["pred3d"][:n, :, :3] = rng.normal([0, 0, 300], [60, 80, 40], (n, 15, 3))
    r["pred3d"][:n, :, 3] = r["pred2d"][:n, :, 3]
    return r


def test_frame_half_is_the_overlay():
    rng = np.random.default_rng(1)
    for h, w in ((240, 320), (300, 121)):
        f = rng.integers(0, 256, (h, w, 3), np.uint8)
        rec = random_record(rng, 6, w, h)
        out = V.render_view3d(f, rec, row(w, h))
        assert out.shape == (h, w + h, 3)
        assert (out[:, :w] == R.render(f, rec, row(w, h))).all()
        assert (out[:, w:] == V.panel(rec, h)).all()


def test_composites_encode_like_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    for h, w, n in ((64, 96, 3), (37, 53, 1), (121, 80, 12)):
        f = rng.integers(0, 256, (h, w, 3), np.uint8)
        img = V.render_view3d(f, random_record(rng, n, w, h), row(w, h))
        ok, b = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), 90])
        assert ok and E.encode(img, 90) == b.tobytes(), (h, w)


def test_cli_vis_3d_arguments(monkeypatch, tmp_path):
    seen = {}

    def fake_run(*a, **k):
        seen.clear()
        seen.update(k)
        return 0

    monkeypatch.setattr(ri, "run", fake_run)
    monkeypatch.setattr(ri, "_load_checkpoints", lambda a: ({}, None))
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_3d", "1"]) == 0
    assert seen["vis_dir"] == "V" and seen["vis_3d"] is True
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_3d", "0"]) == 0
    assert "vis_3d" not in seen, "without --vis_3d, run() is called as before"
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V"]) == 0
    assert "vis_3d" not in seen
    with pytest.raises(SystemExit):
        ri.main(["--output_dir", str(tmp_path), "--vis_3d", "1"])
    with pytest.raises(SystemExit):
        ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_3d", "2"])


def test_a_frame_too_wide_for_the_composite_is_named(tmp_path):
    class NoEncoder:
        def encode_jpeg(self, *a, **k):
            raise AssertionError("encoded")

    frames = [np.zeros((8, 8, 3), np.uint8), np.zeros((100, 16285, 3), np.uint8)]
    with pytest.raises(ValueError, match="wide.jpg is 16285x100"):
        ri.write_vis(NoEncoder(), str(tmp_path), 95, ["a.jpg", "wide.jpg"], frames, None, None, True)


def test_panel_kernels_do_not_spill():
    """nvcc -Xptxas -v on view3d.cu: its 2 kernels use no local memory for spills."""
    import shutil
    import subprocess
    import tempfile

    from smap_b200 import build

    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run(["nvcc"] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "view3d.cu"),
                            "-o", os.path.join(tmp, "v.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    spills = [line for line in p.stdout.splitlines() if "spill" in line]
    assert len(spills) == 2 and all(" 0 bytes spill stores, 0 bytes spill loads" in s for s in spills), p.stdout
