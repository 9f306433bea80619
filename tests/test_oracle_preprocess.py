"""CPU: the pre-processing oracle against (1) digests of the unmodified reference pipeline's outputs
(tests/golden/preprocess_digests.json, written by tests/golden/make_golden.py from dataset/custom_dataset.py +
torchvision) and (2) cv2.resize itself when opencv is importable (it is a third-party dependency of the reference)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import (PRE_GEOMS, RESIZE_KINDS, RESIZE_NETS, cv2_preprocess, preprocess_case_image, resize_geoms,  # noqa: E402
                   resize_image, resize_refused)

from oracle import preprocess_numpy as P  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("ci", range(len(PRE_GEOMS)))
def test_oracle_reproduces_reference_pipeline_digest(ci):
    g = json.load(open(os.path.join(GOLD, "preprocess_digests.json")))["c%d" % ci]
    img = preprocess_case_image(ci)
    assert [img.shape[1], img.shape[0]] == g["geom"]
    u8, _ = P.aug_croppad(img)
    assert hashlib.sha256(np.ascontiguousarray(u8).tobytes()).hexdigest() == g["u8_sha256"]
    t, sc = P.preprocess(img)
    assert t.shape == (3, 512, 832) and t.dtype == np.float32
    assert hashlib.sha256(t.tobytes()).hexdigest() == g["sha256"]
    for k, v in g["scale"].items():
        assert float(sc[k]) == v


def test_value_level_fixture():
    f = np.load(os.path.join(GOLD, "preprocess_small.npz"))
    t, _ = P.preprocess(preprocess_case_image(int(f["ci"])))
    assert np.array_equal(t[:, ::4, ::4], f["tensor"])


def test_resize_against_cv2_when_available():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for (W, H) in [(1920, 1080), (700, 933), (1664, 1024), (64, 40), (832, 512), (1234, 777)]:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        s = min(832 / W, 512 / H)
        assert np.array_equal(cv2.resize(img, (0, 0), fx=s, fy=s), P.resize_linear_u8(img, s))


@pytest.mark.parametrize("kind", RESIZE_KINDS)
def test_oracle_equals_cv2_resize_in_every_regime(kind):
    """resize_linear_u8 against cv2.resize at 832x512 on resize_geoms(): exact 1/2 scale at every parity of W and H mod 4
    (windows cut by an odd last column or row), identity, up-scaling from 1-pixel sides, one-pixel results, 1/3 and 1/4,
    random sizes (noise only); geometries cv2 refuses are refused.  The whole oracle pipeline equals the cv2 reference of
    tests/golden/cases.py, scale dict included."""
    cv2 = pytest.importorskip("cv2")
    geoms = resize_geoms(n_random=None if kind == "noise" else 0)
    for i, (W, H) in enumerate(geoms):
        img = resize_image(kind, W, H, i)
        s = min(832 / W, 512 / H)
        if resize_refused(W, H):
            with pytest.raises(cv2.error):
                cv2.resize(img, (0, 0), fx=s, fy=s)
            with pytest.raises(ValueError):
                P.resize_linear_u8(img, s)
            continue
        want = cv2.resize(img, (0, 0), fx=s, fy=s)
        got = P.resize_linear_u8(img, s)
        assert got.shape == want.shape, (W, H, kind)
        diff = np.argwhere((got != want).any(-1))
        assert len(diff) == 0, (W, H, kind, "%d pixels differ, first at %s" % (len(diff), diff[:3].tolist()))
        if kind != "noise":  # letterbox, normalisation and scale dict at every non-random geometry
            t, sc = P.preprocess(img)
            tr, scr = cv2_preprocess(img)
            assert np.array_equal(t, tr) and sc == scr, (W, H, kind)


def debug_resize_plan(W, H, net_w, net_h):
    """smapb_debug_resize_plan (host only) -> (rc, dims6, scale, xofs, xcoef, yofs, ycoef)."""
    import ctypes

    from smap_b200 import _lib

    fn = _lib.load().smapb_debug_resize_plan
    fn.argtypes = [ctypes.c_int] * 4 + [ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_double), ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    dims = (ctypes.c_int * 6)()
    sc = ctypes.c_double()
    xo = np.zeros(net_w, np.int32); xc = np.zeros(net_w * 2, np.int16); yo = np.zeros(net_h * 2, np.int32); yc = np.zeros(net_h * 2, np.int16)
    rc = fn(W, H, net_w, net_h, dims, ctypes.byref(sc), xo.ctypes.data, xc.ctypes.data, yo.ctypes.data, yc.ctypes.data)
    return rc, list(dims), sc.value, xo, xc, yo, yc


def test_library_accepts_exactly_what_cv2_resize_accepts():
    """make_resize_plan (smapb_debug_resize_plan, the rule smapb_preprocess applies) accepts sides 1 to 16384 and refuses
    exactly where cv2.resize raises (a resized side rounds to 0), at every network size of the sweep; the accepted plans
    have cv2's output size.  Sides above 16384 are a library limit (cv2 takes them)."""
    cv2 = pytest.importorskip("cv2")
    for net_w, net_h in RESIZE_NETS:
        for (W, H) in resize_geoms(net_w, net_h, n_random=0) + [(16384, 16384), (1, 16384), (16384, 1)]:
            s = min(net_w / W, net_h / H)
            try:
                want = cv2.resize(np.zeros((H, W, 3), np.uint8), (0, 0), fx=s, fy=s).shape[:2]
            except cv2.error:
                want = None
            assert (want is None) == resize_refused(W, H, net_w, net_h), (W, H, net_w, net_h)
            rc, dims = debug_resize_plan(W, H, net_w, net_h)[:2]
            if want is None:
                assert rc == -1, ("accepted", W, H, net_w, net_h)
            else:
                assert rc == 0 and (dims[1], dims[0]) == want, (W, H, net_w, net_h, dims, want)
    for (W, H) in [(1, 1), (1, 2), (2, 1), (17, 16384), (16384, 16)]:
        assert debug_resize_plan(W, H, 832, 512)[0] == 0, (W, H)
    for (W, H) in [(2, 16384), (16, 16384), (16384, 9), (1, 1024), (0, 5), (5, 0), (-1, 5), (16385, 16), (16, 16385)]:
        assert debug_resize_plan(W, H, 832, 512)[0] == -1, (W, H)


def test_library_resize_plan_equals_oracle_tables_over_many_geometries():
    """The host-side table builder inside libsmap_b200.so (make_resize_plan) against the oracle's tables - no GPU needed.
    Sweeps 400 source geometries incl. up-scaling, exact 1/2 and 1/1 scales and extreme aspect ratios at 832x512, and
    the resize sweep's geometries at every network size it runs at."""
    rng = np.random.default_rng(77)
    geoms = [(1920, 1080), (1664, 1024), (832, 512), (416, 256), (3328, 2048), (2, 2), (16384, 16384), (5000, 40), (40, 5000)]
    geoms += [(int(rng.integers(8, 4200)), int(rng.integers(8, 3200))) for _ in range(391)]
    cases = [(g, (832, 512)) for g in geoms]
    cases += [(g, net) for net in RESIZE_NETS for g in resize_geoms(*net, n_random=0) if not resize_refused(*g, *net)]
    for (W, H), (net_w, net_h) in cases:
        rc, dims, sc, xo, xc, yo, yc = debug_resize_plan(W, H, net_w, net_h)
        assert rc == 0, (W, H, net_w, net_h)
        s = min(net_w / W, net_h / H)
        assert sc == s
        dw, dh = P.cv_round(W * s), P.cv_round(H * s)
        assert (dims[0], dims[1]) == (dw, dh), (W, H)
        inv = 1.0 / s
        mode = 2 if (dw, dh) == (W, H) else (1 if int(inv) == 2 and abs(2 - inv) < np.finfo(np.float64).eps else 0)
        assert dims[4] == mode, (W, H)
        pad_l = (net_w - dw) // 2 if dw < net_w else 0
        pad_t = (net_h - dh) // 2 if (dw >= net_w and dh < net_h) else 0
        assert (dims[2], dims[3]) == (pad_l, pad_t), (W, H)
        if mode != 0:
            continue
        oxo, oxa = P.linear_tables(W, dw, s)
        assert np.array_equal(xo[:dw], oxo) and np.array_equal(xc[:2 * dw].reshape(dw, 2), oxa), (W, H)
        # vertical taps: clamped rows, unsnapped weights (oracle/preprocess_numpy.py resize_linear_u8)
        for d in range(dh):
            f = np.float32((d + 0.5) * inv - 0.5)
            sy = int(np.floor(f))
            f = np.float32(f - np.float32(sy))
            assert yo[2 * d] == min(max(sy, 0), H - 1) and yo[2 * d + 1] == min(max(sy + 1, 0), H - 1), (W, H, d)
            assert yc[2 * d] == P.cv_round(float(np.float32((np.float32(1.0) - f) * np.float32(2048)))), (W, H, d)
            assert yc[2 * d + 1] == P.cv_round(float(np.float32(f * np.float32(2048)))), (W, H, d)
