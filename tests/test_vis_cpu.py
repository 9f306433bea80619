"""CPU: the skeleton overlay oracle (oracle/render_numpy.py) on hand-built cases, and run_inference --vis_dir's host
logic (argument parsing, output names, collisions)."""
import numpy as np
import pytest

from oracle import render_numpy as R
from smap_b200 import run_inference as ri

RECORD_DTYPE = np.dtype([("pred3d", "<f8", (127, 15, 4)), ("root_depth", "<f8", (127,)), ("pred2d", "<f4", (127, 15, 4)),
                         ("count", "<i4"), ("pad_", "<i4")])


def record(persons):
    """persons: list of {joint: (x, y)} in net-input pixels (score 1)."""
    r = np.zeros((), RECORD_DTYPE)
    r["count"] = len(persons)
    for p, joints in enumerate(persons):
        for j, (x, y) in joints.items():
            r["pred2d"][p, j] = (x, y, 0, 1)
    return r


def row(w, h, nw=832, nh=512):
    s = min(nw / w, nh / h)
    return np.array([s, w, h, nw, nh, w, w, w / 2, h / 2])


def test_horizontal_limb_pixels():
    # a 832x512 frame: scale 1, no letterbox; head (1) to neck (0) from x=100 to x=140 on row 50; r = 1, R = 2
    f = np.zeros((512, 832, 3), np.uint8)
    out = R.render(f, record([{0: (100, 50), 1: (140, 50)}]), row(832, 512))
    assert R.radii(512, 832) == (1, 2)
    limb = np.zeros((512, 832), bool)
    limb[49:52, 100:141] = True  # |y - 50| <= 1 between the endpoints
    limb[50, 99] = limb[50, 141] = True  # the endpoint discs of radius 1
    joints = np.zeros((512, 832), bool)
    for cx in (100, 140):
        yy, xx = np.mgrid[0:512, 0:832]
        joints |= (xx - cx) ** 2 + (yy - 50) ** 2 <= 4
    assert (out[joints] == 255).all()
    assert (out[limb & ~joints] == (0, 0, 255)).all()
    assert (out[~limb & ~joints] == 0).all()


def test_later_persons_paint_over_earlier_ones():
    f = np.zeros((512, 832, 3), np.uint8)
    a = {3: (200, 200), 4: (260, 200)}
    b = {3: (230, 170), 4: (230, 230)}
    out = R.render(f, record([a, b]), row(832, 512))
    assert (out[200, 230] == (0, 255, 0)).all(), "the crossing takes the later person's colour"
    assert (out[185, 230] == (0, 255, 0)).all(), "person 1's vertical limb over person 0's horizontal one"
    assert (out[200, 215] == (0, 0, 255)).all()


def test_zero_score_joints_and_their_limbs_are_skipped():
    f = np.zeros((512, 832, 3), np.uint8)
    r = record([{0: (100, 50), 1: (140, 50)}])
    r["pred2d"][0, 1, 3] = 0
    out = R.render(f, r, row(832, 512))
    assert (out[50, 120] == 0).all(), "no limb to a joint with score 0"
    assert (out[50, 140] == 0).all() and (out[50, 100] == 255).all()
    assert (R.render(f, record([]), row(832, 512)) == f).all()


@pytest.mark.parametrize("w,h", [(1000, 1000), (2000, 600)])
def test_letterbox_on_each_axis(w, h):
    s, pad_l, pad_t = R.letterbox(row(w, h))
    if w == 1000:
        assert pad_l == (832 - round(1000 * s)) // 2 and pad_l > 0 and pad_t == 0
    else:
        assert pad_t == (512 - round(600 * s)) // 2 and pad_t > 0 and pad_l == 0
    x, y = pad_l + 100 * s, pad_t + 50 * s  # frame pixel (100, 50)
    pts = R.joints(record([{2: (x, y)}]), row(w, h))
    assert pts[0][2] == (100, 50)
    f = np.zeros((h, w, 3), np.uint8)
    out = R.render(f, record([{2: (x, y)}]), row(w, h))
    assert (out[50, 100] == 255).all()


def test_coordinates_outside_the_frame():
    f = np.zeros((512, 832, 3), np.uint8)
    # a limb from far outside the left edge into the frame, and a joint off the bottom
    out = R.render(f, record([{0: (-5000, 100), 9: (50, 100), 14: (400, 900)}]), row(832, 512))
    assert (out[100, 0:45] == (0, 0, 255)).all()
    assert (out[500:, :] == 0).all()
    pts = R.joints(record([{0: (1e9, -1e9)}]), row(832, 512))
    assert pts[0][0] == (R.COORD_MAX, -R.COORD_MAX)


def test_vis_names_and_collisions():
    paths = ["/d/a.png", "/d/sub/b.jpeg", "/d/c.jpg"]
    assert ri.vis_names(paths, "/d") == ["a.jpg", "sub/b.jpg", "c.jpg"]
    with pytest.raises(ValueError, match="/d/a.png and /d/a.jpg"):
        ri.vis_names(["/d/a.png", "/d/a.jpg"], "/d")


def test_cli_arguments(monkeypatch, tmp_path):
    seen = {}

    def fake_run(*a, **k):
        seen.update(k)
        return 0

    monkeypatch.setattr(ri, "run", fake_run)
    monkeypatch.setattr(ri, "_load_checkpoints", lambda a: ({}, None))
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_quality", "80"]) == 0
    assert seen["vis_dir"] == "V" and seen["vis_quality"] == 80
    seen.clear()
    assert ri.main(["--output_dir", str(tmp_path)]) == 0
    assert "vis_dir" not in seen and "vis_quality" not in seen, "without --vis_dir, run() is called as before"
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V"]) == 0
    assert seen["vis_quality"] == 95
    with pytest.raises(SystemExit):
        ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_quality", "0"])


def test_collision_is_refused_before_any_work(tmp_path, monkeypatch):
    (tmp_path / "a.png").write_bytes(b"x")
    (tmp_path / "a.jpg").write_bytes(b"x")

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(ri, "Engine", no_engine)
    with pytest.raises(ValueError, match="a.jpg"):
        ri.run({}, str(tmp_path), str(tmp_path / "o.json"), vis_dir=str(tmp_path / "v"))
