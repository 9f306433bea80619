"""GPU: the association kernels at map sizes other than 128x208, bit for bit against the live reference and the oracle,
on the adversarial frames of tests/golden/assoc_adversary.py built at each size.

The kernels take the map size at run time, and other sizes run other kernel instances: the scalar NMS flag kernel
(`nms_flag_kernel<false>`, h*w % 128 != 0) and the PAF kernel that gathers from global memory (`paf_kernel<false>`, both
planes above 227 KB of shared memory, h*w > 28 798).  The near threshold sqrtf(h*w)/150, border and window clipping and
the root-depth reads move with the size.  tests/test_assoc_reference_gpu.py sees none of this: it runs at 128x208 only.

oracle/build_ref.py builds dapalib_ref_dims, the unmodified reference sources plus our map-size setter
(oracle/ref_map_size.cpp).  The setter refuses the sizes at which the reference's NMS is not deterministic (w % 16 != 0:
racing border writes; h*w % 512 != 0: a divergent __syncthreads()); those sizes are compared with the oracle alone, and
this file checks that the setter refuses them without running the reference there.  The scalar flag kernel can never
meet the live reference (h*w % 512 == 0 implies h*w % 128 == 0): the oracle, pinned to the live reference at every
allowed size here, is its only check.

At every size, with one Engine(0, B, 4h, 4w) handle per size:
  * Engine.extract: peak counts, peaks, the nA x nB score blocks and the dense -1 fill around them;
  * Engine.connect: roots 0 and 2, dist_flag on and off;
  * oracle.assoc.extract / connect equal the kernels everywhere and the live reference where the size allows it;
  * Engine.lift on the connected bodies, and on bodies with joints on the last map row and column, equals lift_numpy.
Values are compared as uint32 bit patterns.  The reference's connect groups with one tensor .item() per pair score
(about a second per 127-person frame), so it runs on a subset of each size's frames (`ref_connects`)."""
import time

import numpy as np
import pytest
import torch

import assoc_adversary as A
from oracle import assoc, build_ref, lift_numpy
from test_assoc_reference_gpu import compare_bodies, compare_extract, diff

pytestmark = pytest.mark.gpu
COMBOS = [(r, d) for r in (0, 2) for d in (True, False)]
MAX_REPORT = 8

# (h, w, live reference, random_heatmaps / make_scene seeds of the breadth family): see DESIGN.md section 5
SIZES = [
    (128, 208, True, 1),    # control: vectorised NMS, staged PAF; the dims module must equal dapalib_ref here
    (8, 64, True, 1),       # 6 interior rows: every centroid window clipped top and bottom
    (256, 16, True, 1),     # 14 interior columns
    (32, 32, True, 1),      # small map: the 127 cap and crowding on a 2 px grid
    (128, 224, True, 1),    # the largest staged PAF size the reference allows (231 440 B of shared memory)
    (152, 192, True, 1),    # the smallest unstaged size the reference allows (235 536 B: global gathers)
    (256, 256, True, 1),    # config 5 (1024x1024 input)
    (120, 240, False, 1),   # first size past staging (16 B over); 28 800 % 512 = 128: oracle only
    (120, 200, False, 1),   # scalar NMS (24 000 % 128 = 64), staged PAF; w % 16 = 8: oracle only
    (360, 1000, False, 0),  # scalar NMS, global PAF, near threshold exactly 4.0f: oracle only
]


def ref_runs(name):
    """Frames the live reference extracts: all but eight of the ten 127-key sets (`equal` and `heap` stay).  The others
    are the same kind of frame, 127 root peaks on noise, and differ in their root depths, which only connect reads."""
    return not (name.startswith("group_keys_") and "_n127" in name and "heap" not in name and "equal" not in name)


def ref_connects(name, root_idx, dist_flag, control=False):
    """Frames the live reference connects (the oracle and the kernels connect every frame).  Root 2 with the penalty:
    every NMS, PAF and grouping frame but the saturated one, one crowded frame and one scene.  The other three
    combinations: the grouping frames (ties, `used`, penalties) and the border and near-threshold frames.  The key-set
    frames connect on the root they were built for, with the penalty.  At the control size only the first combination:
    tests/test_assoc_reference_gpu.py runs all four there."""
    if not ref_runs(name) or control and (root_idx, dist_flag) != (2, True):  # see the docstring
        return False
    if name.startswith("group_keys_"):
        return name.endswith("root%d" % root_idx) and dist_flag
    if (root_idx, dist_flag) == (2, True):
        return name.startswith(("nms_", "paf_", "group_")) and name != "nms_saturated" or \
            name in ("crowded_0", "scene_0")
    return name.startswith(("group_", "paf_near", "nms_border"))


def size_frames(h, w, seeds):
    yield from A.frames(h, w, families=("nms", "paf", "group"))
    yield from A.breadth_frames(h, w, seeds)


@pytest.fixture(scope="module")
def ref_dims():
    r = build_ref.load_ref_dims()
    if r is None:
        pytest.skip("oracle/_ref/dims/dapalib_ref_dims*.so is missing: build() builds it where the reference sources "
                    "exist")
    return r


def sync():
    torch.cuda.synchronize()


def ref_extract(mod, hms):
    th = torch.from_numpy(hms).cuda().contiguous()  # exactly [43, h, w] float32: the reference copies that many
    assert th.dtype == torch.float32 and th.is_contiguous()
    sync()
    pk, sc = mod.extract(th)
    sync()
    return [p.numpy().copy() for p in pk], [s.numpy().copy() for s in sc]


def ref_connect(mod, hms, rd, root_idx, dist_flag):
    assert A.connectable(hms, root_idx)
    th = torch.from_numpy(hms).cuda().contiguous()
    sync()
    b = mod.connect(th, torch.from_numpy(rd).contiguous(), root_idx, dist_flag)  # depth map on the CPU
    sync()
    b = b.numpy().copy()
    return b if b.ndim == 3 else np.zeros((0, A.NJ, 4), np.float32)


def dense_fill(name, peaks, scores):
    """Outside the nA x nB block every score is -1 (pafScoreKernel writes it for every pair it does not score)."""
    for l in range(A.NL):
        na, nb = int(peaks[A.PAIRS[2 * l], 0, 0]), int(peaks[A.PAIRS[2 * l + 1], 0, 0])
        m = np.ones((A.MAXP, A.MAXP), bool)
        m[:na, :nb] = False
        if not (scores[l][m].view(np.uint32) == np.float32(-1).view(np.uint32)).all():
            return "%s limb %d: a score outside the %d x %d block is not -1" % (name, l, na, nb)
    return None


def chunks(gen, n):
    buf = []
    for f in gen:
        buf.append(f)
        if len(buf) == n:
            yield buf
            buf = []
    if buf:
        yield buf


def lift_inputs(h, w, n, seed):
    """det_d [n,14,h,w], a scale row per frame for a 4w x 4h network input of a 2x larger image."""
    rng = np.random.default_rng(seed)
    dd = (rng.normal(0, 20, (n, A.NL, h, w))).astype(np.float32)
    sc = lift_numpy.default_scale(8 * w, 8 * h, net_w=4 * w, net_h=4 * h)
    from smap_b200.engine import scale_row

    return dd, sc, np.stack([scale_row(sc)] * n)


def edge_bodies(h, w, P, seed):
    """[P,15,4] bodies as connect returns them, with joints on the last map row and column (x = w - 0.5, y = h - 0.5)
    and on the first (0.5), every person with a root."""
    rng = np.random.default_rng(seed)
    b = np.zeros((P, A.NJ, 4), np.float32)
    b[:, :, 0] = rng.uniform(0.5, w - 0.5, (P, A.NJ))
    b[:, :, 1] = rng.uniform(0.5, h - 0.5, (P, A.NJ))
    b[:, :, 0][rng.uniform(size=(P, A.NJ)) < 0.2] = w - 0.5
    b[:, :, 1][rng.uniform(size=(P, A.NJ)) < 0.2] = h - 0.5
    b[:, :, 0][rng.uniform(size=(P, A.NJ)) < 0.05] = 0.5
    b[:, :, 1][rng.uniform(size=(P, A.NJ)) < 0.05] = 0.5
    b[:, :, 3] = rng.uniform(0.2, 1, (P, A.NJ)) * (rng.uniform(size=(P, A.NJ)) > 0.25)
    b[:, 2, 3] = rng.uniform(0.2, 1, P)
    b[b[:, :, 3] == 0] = 0
    return b


def check_lift(eng, bodies, counts, dd, rd, sc, scales, names):
    """Engine.lift on device bodies/counts against lift_numpy on the same bodies: pred2d and root depths bit for bit,
    pred3d within 1e-12 (float64, as in tests/test_assoc_limits_gpu.py), NaN where lift_numpy has NaN (NaN root
    depths of the key-set frames)."""
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    p2, p3, rdp, co = eng.lift(dev(bodies), dev(counts), dev(dd), dev(rd), dev(scales))
    sync()
    p2, p3, rdp, co = p2.cpu().numpy(), p3.cpu().numpy(), rdp.cpu().numpy(), co.cpu().numpy()
    errs = []
    for b, name in enumerate(names):
        o2, o3, ordp = lift_numpy.lift(bodies[b, :int(counts[b])], dd[b], rd[b], sc)
        m = len(o2)
        e = None
        if int(co[b]) != m:
            e = "%s lift: %d persons, lift_numpy %d" % (name, int(co[b]), m)
        else:
            e = diff(p2[b, :m], o2, "%s lift pred2d" % name)
            same = np.array_equal(rdp[b, :m].view(np.uint64), np.asarray(ordp, np.float64).view(np.uint64))
            if e is None and not same:
                e = "%s lift root depths differ" % name
            if e is None and not np.allclose(p3[b, :m], o3, rtol=1e-12, atol=1e-12, equal_nan=True):  # NaN depths
                e = "%s lift pred3d differs by %g" % (name, float(np.nanmax(np.abs(p3[b, :m] - o3))))
            if e is None and (p2[b, m:].any() or p3[b, m:].any()):
                e = "%s lift: rows past the count are not zero" % name
        if e:
            errs.append(e)
    return errs


@pytest.mark.parametrize("h,w,live,seeds", SIZES, ids=["%dx%d" % s[:2] for s in SIZES])
def test_association_at_size(ref_dims, h, w, live, seeds):
    from smap_b200.engine import Engine

    mod, set_size = ref_dims
    rc = set_size(h, w)
    if not live:  # refused by the setter: the reference never runs here
        assert rc != 0 and set_size.get() != (h, w), "the setter accepted %dx%d" % (h, w)
    else:
        assert rc == 0 and set_size.get() == (h, w)
    t0 = time.time()
    free0 = torch.cuda.mem_get_info()[0]
    batch = 4 if h * w > 256 * 256 else 8
    eng = Engine(0, max_batch=batch, in_h=4 * h, in_w=4 * w)
    sync()
    t_setup, mem = time.time() - t0, free0 - torch.cuda.mem_get_info()[0]
    errs = {k: [] for k in ("extract", "oracle extract", "kernel vs oracle", "connect", "oracle connect", "lift")}
    n_ext = n_conn = n_ref_ext = n_ref_conn = n_lift = 0
    t_ref_ext = t_ref_conn = 0.0
    try:
        for chunk in chunks(size_frames(h, w, seeds), batch):
            names = [f[0] for f in chunk]
            hms = np.stack([f[1] for f in chunk])
            rds = np.stack([f[2] for f in chunk])
            hd, rdd = torch.from_numpy(hms).cuda(), torch.from_numpy(rds).cuda()
            sync()
            p, s = eng.extract(hd)
            sync()
            p, s = p.cpu().numpy(), s.cpu().numpy()
            for b, name in enumerate(names):
                n_ext += 1
                op, os_ = assoc.extract(hms[b])
                e = (diff(p[b], op, "%s peaks" % name) or diff(s[b], os_, "%s scores" % name) or
                     dense_fill(name, p[b], s[b]))
                if e:
                    errs["kernel vs oracle"].append(e)
                if live and ref_runs(name):
                    n_ref_ext += 1
                    t = time.time()
                    want = ref_extract(mod, hms[b])
                    t_ref_ext += time.time() - t
                    e = compare_extract(name, p[b], s[b], want)
                    if e:
                        errs["extract"].append(e)
                    e = compare_extract("oracle " + name, op, os_, want)
                    if e:
                        errs["oracle extract"].append(e)
            ok = [b for b, f in enumerate(chunk) if "extract_only" not in f[3]]  # +-inf in a root plane
            chunk, names, hms, rds = [chunk[b] for b in ok], [names[b] for b in ok], hms[ok], rds[ok]
            hd, rdd = torch.from_numpy(hms).cuda(), torch.from_numpy(rds).cuda()
            for root_idx, dist_flag in COMBOS:
                bodies, counts = eng.connect(hd, rdd, root_idx, dist_flag)
                sync()
                bodies_h, counts_h = bodies.cpu().numpy(), counts.cpu().numpy()
                for b in range(len(chunk)):
                    name = "%s root %d dist %s" % (names[b], root_idx, dist_flag)
                    n_conn += 1
                    ob = assoc.connect(hms[b], rds[b], root_idx, dist_flag)
                    e = compare_bodies("kernel vs oracle " + name, bodies_h[b], int(counts_h[b]), ob)
                    if e:
                        errs["kernel vs oracle"].append(e)
                    control = (h, w) == (A.H, A.W)
                    if live and ref_connects(names[b], root_idx, dist_flag, control) and A.connectable(hms[b], root_idx):
                        n_ref_conn += 1
                        t = time.time()
                        want = ref_connect(mod, hms[b], rds[b], root_idx, dist_flag)
                        t_ref_conn += time.time() - t
                        e = compare_bodies(name, bodies_h[b], int(counts_h[b]), want)
                        if e:
                            errs["connect"].append(e)
                        e = compare_bodies("oracle " + name,
                                           np.concatenate([ob, np.zeros((1, A.NJ, 4), np.float32)]), len(ob), want)
                        if e:
                            errs["oracle connect"].append(e)
                if (root_idx, dist_flag) == (2, True):  # the lift on the connected bodies of the frames
                    dd, sc, scales = lift_inputs(h, w, len(chunk), n_ext)
                    errs["lift"] += check_lift(eng, bodies_h, counts_h, dd, rds, sc, scales, names)
                    n_lift += len(chunk)
        # the lift with joints on the last map row and column: 127 and 19 persons
        P = np.array([A.MAXP, 19], np.int32)
        bodies = np.zeros((2, A.MAXP, A.NJ, 4), np.float32)
        for i, n in enumerate(P):
            bodies[i, :n] = edge_bodies(h, w, n, 40 + i)
        dd, sc, scales = lift_inputs(h, w, 2, 99)
        rds = np.random.default_rng(98).uniform(1, 9, (2, h, w)).astype(np.float32)
        errs["lift"] += check_lift(eng, bodies, P, dd, rds, sc, scales, ["edge_bodies_%d" % n for n in P])
        assert (bodies[:, :, :, 0] == w - 0.5).any() and (bodies[:, :, :, 1] == h - 0.5).any()
        n_lift += 2
    finally:
        eng.close()
        if live:
            set_size(A.H, A.W)
    print("\n%dx%d (%s): extract %d frames (%d against the live reference), connect %d frame-combos (%d), lift %d "
          "frames; the reference's extract %.1f s, its connect %.1f s; handle set-up %.2f s, %.0f MB; wall %.1f s"
          % (h, w, "live reference + oracle" if live else "oracle only", n_ext, n_ref_ext, n_conn, n_ref_conn, n_lift,
             t_ref_ext, t_ref_conn, t_setup, mem / 2 ** 20, time.time() - t0))
    left = sorted(k[2] for k in A.LEFT_OUT if k[:2] == (h, w))
    if left:
        print("  left out at this size: " + ", ".join(left))
    assert n_ext > 0 and n_conn > 0 and (n_ref_conn > 0 or not live)
    bad = ["%s: %d differ\n    %s" % (k, len(v), "\n    ".join(v[:MAX_REPORT])) for k, v in errs.items() if v]
    if bad:
        pytest.fail("%dx%d:\n  " % (h, w) + "\n  ".join(bad))


def test_dims_module_equals_the_plain_reference_at_128x208(ref_dims):
    """At 128x208 the reference with our setter linked in returns exactly what dapalib_ref returns (the module the
    recorded assoc_ref.npz and tests/test_assoc_reference_gpu.py use): the second build changes nothing but the size."""
    plain = build_ref.load_ref()
    if plain is None:
        pytest.skip("oracle/_ref/dapalib_ref*.so is missing")
    mod, set_size = ref_dims
    assert set_size(A.H, A.W) == 0
    n = 0
    for name, hms, rd, targets in A.frames(families=("nms", "paf")):
        a, b = ref_extract(mod, hms), ref_extract(plain, hms)
        assert [x.shape for x in a[0]] == [x.shape for x in b[0]], name
        for x, y in zip(a[0] + a[1], b[0] + b[1]):
            assert diff(x, y, name) is None, diff(x, y, name)
        if "extract_only" not in targets and name.startswith("nms_cap"):
            assert diff(ref_connect(mod, hms, rd, 2, True), ref_connect(plain, hms, rd, 2, True), name) is None
        n += 1
    assert n > 15
