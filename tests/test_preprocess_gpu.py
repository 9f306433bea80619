"""GPU: smapb_preprocess / smapb_preprocess_host (SURVEY 8(f) f1) against the oracle and the reference digests, and against
cv2.resize itself over a sweep of geometries at five network sizes: bit-exact."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from cases import (PRE_GEOMS, RESIZE_NETS, cv2_preprocess, preprocess_case_image, resize_geoms, resize_image,  # noqa: E402
                   resize_refused)

from oracle import preprocess_numpy as P  # noqa: E402
from smap_b200.engine import scale_row  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=4, in_h=512, in_w=832)
    yield e
    e.close()


def test_all_reference_geometries_bit_exact(eng):
    gold = json.load(open(os.path.join(GOLD, "preprocess_digests.json")))
    imgs = [preprocess_case_image(ci) for ci in range(len(PRE_GEOMS))]
    for lo in range(0, len(imgs), 4):
        chunk = imgs[lo:lo + 4]
        # alternate device-resident and host images: both entry points
        feed = [torch.from_numpy(im).cuda() if (lo + i) % 2 == 0 else im for i, im in enumerate(chunk)]
        out, scales = eng.preprocess(feed)
        out = out.cpu().numpy()
        for i, im in enumerate(chunk):
            ci = lo + i
            want, sc = P.preprocess(im)
            assert np.array_equal(out[i], want), "geometry %s differs from the oracle" % (PRE_GEOMS[ci],)
            assert hashlib.sha256(np.ascontiguousarray(out[i]).tobytes()).hexdigest() == gold["c%d" % ci]["sha256"]
            assert np.array_equal(scales[i].numpy(), scale_row(sc))


def test_same_geometry_reuses_tables_and_random_noise(eng):
    rng = np.random.default_rng(9)
    for _ in range(3):
        im = rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
        out, _ = eng.preprocess([torch.from_numpy(im).cuda()])
        assert np.array_equal(out[0].cpu().numpy(), P.preprocess(im)[0])


def check_against_cv2(eng, geoms, kinds, alt=0):
    """Engine.preprocess of each (W, H) x kind image, device and host images alternating, against cv2.resize + letterbox +
    normalise (cases.cv2_preprocess): bit for bit, scale row included.  Geometries cv2 refuses raise SmapB200Error
    naming the geometry.  -> number of images checked."""
    pytest.importorskip("cv2")
    from smap_b200.engine import SmapB200Error

    n = 0
    for i, (W, H) in enumerate(geoms):
        for kind in kinds:
            im = resize_image(kind, W, H, i)
            feed = torch.from_numpy(im).cuda() if (n + alt) % 2 == 0 else im
            n += 1
            if resize_refused(W, H, eng.in_w, eng.in_h):
                with pytest.raises(SmapB200Error, match="a %dx%d image" % (W, H)):
                    eng.preprocess([feed])
                continue
            out, scales = eng.preprocess([feed])
            want, sc = cv2_preprocess(im, eng.in_w, eng.in_h)
            got = out[0].cpu().numpy()
            bad = np.argwhere((got != want).any(0))
            assert len(bad) == 0, ((eng.in_w, eng.in_h), (W, H), kind, "device" if torch.is_tensor(feed) else "host",
                                   "%d pixels differ, first at (y, x) %s" % (len(bad), bad[:3].tolist()))
            assert np.array_equal(scales[0].numpy(), scale_row(sc)), ((W, H), scales[0], sc)
    return n


def test_resize_sweep_equals_cv2_past_the_plan_cache():
    """832x512 on one handle: the resize sweep (every parity of W and H mod 4 at exact 1/2 scale, 1-pixel sides, one-pixel
    results, 1/3 and 1/4, random sizes) with noise, and its non-random geometries with checkerboards and flat 255.  More
    than 256 distinct geometries pass through the handle, so its plan cache drops everything at least once; the first
    geometries are checked again after that, device and host swapped."""
    from smap_b200.engine import Engine

    geoms = resize_geoms()
    assert sum(not resize_refused(W, H) for W, H in geoms) > 256
    e = Engine(0, max_batch=1, in_h=512, in_w=832)
    try:
        check_against_cv2(e, geoms, ("noise",))
        check_against_cv2(e, resize_geoms(n_random=0), ("check", "flat"))
        check_against_cv2(e, geoms[:24], ("noise",), alt=1)
    finally:
        e.close()


@pytest.mark.parametrize("net", RESIZE_NETS[1:], ids=lambda n: "%dx%d" % n)
def test_resize_sweep_equals_cv2_at_other_network_sizes(net):
    """The same sweep into 1024x1024 (config 5), 96x64, 992x32 and 32x1024 inputs, with the half-scale parity cases of
    each size (e.g. 2047x2048 and 2048x2047 into 1024x1024, 1983x64 and 1984x63 into 992x32)."""
    from smap_b200.engine import Engine

    net_w, net_h = net
    e = Engine(0, max_batch=1, in_h=net_h, in_w=net_w)
    try:
        check_against_cv2(e, resize_geoms(net_w, net_h, n_random=20), ("noise",))
        check_against_cv2(e, resize_geoms(net_w, net_h, n_random=0), ("check", "flat"), alt=1)
    finally:
        e.close()


def test_host_staging_grows_and_is_reused():
    """Host images on a fresh handle: large, small, the large one again, then a larger one (the staging buffer is
    reallocated); each equals the cv2 reference."""
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=1, in_h=512, in_w=832)
    try:
        for (W, H), seed in [((1663, 1024), 1), ((3, 1024), 2), ((1663, 1024), 3), ((2600, 1999), 4), ((1, 1), 5)]:
            im = resize_image("noise", W, H, seed)
            out, scales = e.preprocess([im])
            want, sc = cv2_preprocess(im)
            assert np.array_equal(out[0].cpu().numpy(), want), (W, H)
            assert np.array_equal(scales[0].numpy(), scale_row(sc))
    finally:
        e.close()


def test_preprocess_feeds_the_whole_path(eng):
    """uint8 frames -> preprocess -> infer_device equals feeding the oracle-preprocessed tensor."""
    from smap_b200 import schema
    from smap_b200.engine import records_to_numpy

    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    ims = [preprocess_case_image(0), preprocess_case_image(5)]
    x, scales = eng.preprocess([torch.from_numpy(i).cuda() for i in ims])
    rec = records_to_numpy(eng.infer_device(x, scales.cuda()))
    xo = torch.from_numpy(np.stack([P.preprocess(i)[0] for i in ims])).cuda()
    so = torch.from_numpy(np.stack([scale_row(P.preprocess(i)[1]) for i in ims])).cuda()
    ref = records_to_numpy(eng.infer_device(xo, so))
    assert rec.tobytes() == ref.tobytes()
