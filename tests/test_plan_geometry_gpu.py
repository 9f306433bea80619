"""GPU: the per-op checker of tests/plan_check.py (check_plan), in bf16x3, bf16 and fp16, at the input geometries and
plan paths no other test builds, and the association at map sizes that take its scalar NMS path.

  * edge geometries (in_h x in_w, B): 32x32 B=2 (deepest level 1x1, flat M = 2), 32x992 B=2 (levels one row high),
    1024x32 B=1 (levels one column wide, 64x2 levels tiled tw = 2), 224x288 B=5 (odd levels 7x9 ... 56x72, ragged flat
    M): every op against its float64 reference, every wrong reference that applies flagged;
  * the fallback plan (SMAPB_STEM=cuda: the CUDA-core stem, which the library also takes when the driver rejects the
    tensor-core stem's overlapped TMA view), checked the same way;
  * plans with B < max_batch on one handle give every op the bits of the same images in the B = max_batch plan;
  * forced tile widths change no bit at the edge geometries;
  * association (extract, connect) bit-exact against the oracle at heat-map sizes with h*w % 128 != 0 (scalar NMS flag
    kernel), with peaks on and next to the border;
  * the whole path (records) against the oracle chain at small geometries, and two handles of different geometry
    alternating in one process.
Coverage assertions (test_edge_and_stem_fallback_plans_cover_what_they_are_for) read the op descriptions, so that this
file cannot quietly stop checking what it is for.  `-s` prints the worst |y - r| / bound per op kind of every checked
plan."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import assoc, lift_numpy, smap_torch
from smap_b200 import schema
from smap_b200.synth import make_scene

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import (SEED, _dims, _gid, assert_checked, check_plan, check_switches, dump, op_class,  # noqa: E402
                        plan_ops, plan_summary)

pytestmark = pytest.mark.gpu

EDGE_GEOMS = [(32, 32, 2), (32, 992, 2), (1024, 32, 1), (224, 288, 5)]  # all in bf16x3
SMALL_GEOMS = [(32, 32, 2), (1024, 32, 1)]  # also in bf16 and fp16
FALLBACKS = {"stem_cuda": ("SMAPB_STEM", "cuda")}
FALLBACK_RUNS = [("bf16x3", (32, 32, 2)), ("fp16", (32, 32, 2)), ("bf16x3", (96, 160, 3)), ("fp16", (96, 160, 3)),
                 ("bf16x3", (512, 832, 2))]


# ---------------------------------------------------------------------------------------------------------------------
# per-op parity
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", EDGE_GEOMS, ids=_gid)
def test_edge_geometry_ops_bf16x3(geom):
    assert_checked(plan_summary("bf16x3", geom), "bf16x3")


@pytest.mark.parametrize("geom", SMALL_GEOMS, ids=_gid)
@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_edge_geometry_ops_bf16_fp16(precision, geom):
    assert_checked(plan_summary(precision, geom), precision)


@pytest.mark.parametrize("precision,geom", FALLBACK_RUNS, ids=["%s_%s" % (p, _gid(g)) for p, g in FALLBACK_RUNS])
@pytest.mark.parametrize("fallback", sorted(FALLBACKS))
def test_fallback_plan_ops(fallback, precision, geom):
    s = plan_summary(precision, geom, FALLBACKS[fallback])
    assert_checked(s, precision)
    ops = s["ops"]
    kinds = {o["kind"] for o in ops}
    # the CUDA-core stem replaces s2d + the tensor-core stem
    assert "stem" in kinds and not kinds & {"stem_tc", "s2d"}, kinds


def test_edge_and_stem_fallback_plans_cover_what_they_are_for():
    """Across this file's checked plans: 1-pixel levels, images smaller than one tile, tw = 2, and the fallback stem."""
    runs = [plan_summary("bf16x3", g) for g in EDGE_GEOMS]
    runs += [plan_summary(p, g) for p in ("bf16", "fp16") for g in SMALL_GEOMS]
    runs += [plan_summary(p, g, FALLBACKS[f]) for f in sorted(FALLBACKS) for p, g in FALLBACK_RUNS]
    seen = set()
    for s in runs:
        ops = s["ops"]
        for o in ops:
            if o["kind"] == "stem":
                seen.add("kind stem")
            if o["kind"] not in ("conv", "conv_f32"):
                continue
            N, H, W, _ = _dims(o)
            src = lambda role: _dims(ops[int(o[role])])[1:3]  # noqa: E731  (H, W) of an input's producer
            flat = o["k"] == "1x1" and o["s"] == "1" and ("in2" not in o or o["s2"] == "1") and "up" not in o
            tw = int(o["tw"])
            if 1 in (H, W):
                seen.add("conv with a 1-pixel output dimension")
            if o["k"] == "3x3" and src("in") == [1, 1]:
                seen.add("3x3 conv on a 1x1 input")
            if op_class(o) == "up_residual" and 1 in src("up"):
                seen.add("up-residual from a 1-pixel level")
            if flat and N * H * W < 128:
                seen.add("flat conv with N*Ho*Wo < 128")
            if not flat and (H < 128 // tw or W < tw):
                seen.add("patch conv on an image smaller than one tile")
            if not flat and tw == 2:
                seen.add("tw = 2")
    need = {"conv with a 1-pixel output dimension", "3x3 conv on a 1x1 input", "up-residual from a 1-pixel level",
            "flat conv with N*Ho*Wo < 128", "patch conv on an image smaller than one tile", "tw = 2", "kind stem"}
    assert need <= seen, "not covered: %s" % sorted(need - seen)


@pytest.mark.parametrize("geom", [(1024, 32, 1), (224, 288, 5)], ids=_gid)
def test_edge_geometry_forced_tile_widths_keep_the_bits(geom, monkeypatch):
    """Every forced tile width (tile table rewritten, autotuner off) gives the bits of the autotuned plan."""
    check_switches(geom, monkeypatch, "bf16x3")


# ---------------------------------------------------------------------------------------------------------------------
# B < max_batch
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


@pytest.mark.parametrize("H,W", [(224, 288), (32, 32)], ids=["224x288", "32x32"])
def test_smaller_batches_give_every_op_the_same_bits(H, W):
    """One handle with max_batch = 5: the B = 1 plan on image 2 and the B = 3 plan on images 1-3 give every op (and the
    returned tensors) the bits of the same images in the B = 5 plan, where a 128-row flat tile spans several images.
    The B = 3 plan is then checked op by op."""
    from smap_b200.engine import Engine

    sd = smap_torch.make_state_dict(SEED, "random")
    x = smap_torch.make_input(5, H, W, seed=SEED + 4).cuda()
    eng = Engine(0, max_batch=5, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, "bf16x3")
        outs5 = [o.clone() for o in eng.forward(x)]
        torch.cuda.synchronize()
        _, ops5 = plan_ops(eng, 5)
        full = [dump(eng, 5, o) for o in ops5]
        for lo, hi in ((2, 3), (1, 4)):
            B = hi - lo
            outs = eng.forward(x[lo:hi])
            torch.cuda.synchronize()
            _, ops = plan_ops(eng, B)
            assert [o["name"] for o in ops] == [o["name"] for o in ops5]
            diff = []
            for o, t5 in zip(ops, full):
                ref = t5[lo:hi] if t5.dtype == torch.float32 else t5[:, lo:hi]
                if not torch.equal(_bits(dump(eng, B, o)), _bits(ref)):
                    diff.append("%d %s" % (o["idx"], o["name"]))
            assert not diff, "B=%d: %d ops differ from the B=5 plan, first %s" % (B, len(diff), diff[:3])
            for a, b in zip(outs, outs5):
                assert torch.equal(_bits(a), _bits(b[lo:hi])), "B=%d: returned tensors differ" % B
        del full
        assert_checked(check_plan("bf16x3", H, W, 3, eng=eng), "bf16x3")
    finally:
        eng.close()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# association on the scalar NMS path
# ---------------------------------------------------------------------------------------------------------------------
ASSOC_SIZES = [(8, 8), (24, 40), (56, 72), (8, 248)]


def _noise(seed, h, w, B=2):
    """Backbone-like garbage as in tests/test_assoc_gpu.py (random_heatmaps) at h x w: many peaks."""
    rng = np.random.default_rng(seed)
    lo = rng.normal(0, 1, (B, 43, h // 4, w // 4)).astype(np.float32)
    hms = np.kron(lo, np.ones((1, 1, 4, 4), np.float32)) * 0.4 + rng.normal(0, 0.15, (B, 43, h, w)).astype(np.float32)
    return hms.astype(np.float32), rng.uniform(0.5, 3, (B, h, w)).astype(np.float32)


def _blob(h, w, y, x):
    yy, xx = np.mgrid[0:h, 0:w]
    return (0.9 * np.exp(-((yy - y) ** 2 + (xx - x) ** 2) / 2.0)).astype(np.float32)


BORDER_BLOBS = [(f, side, d) for f, sides in ((0, ("top", "left")), (1, ("bottom", "right"))) for side in sides
                for d in range(4)]


def _border(h, w):
    """One Gaussian blob per keypoint channel, centred on a border row or column (d = 0: excluded by the 3x3 border rule,
    and its neighbours are not maxima) or d = 1..3 pixels from it (a peak whose 7x7 centroid window is clipped).
    Frame 0: top rows (channels 0-3), left columns (4-7); frame 1: bottom rows, right columns."""
    hms = np.zeros((2, 43, h, w), np.float32)
    for f, side, d in BORDER_BLOBS:
        c = d + (4 if side in ("left", "right") else 0)
        y = {"top": d, "bottom": h - 1 - d}.get(side, h // 2)
        x = {"left": d, "right": w - 1 - d}.get(side, w // 2)
        hms[f, c] = _blob(h, w, y, x)
    return hms, np.full((2, h, w), 1.5, np.float32)


def assoc_inputs(h, w):
    persons = max(1, min(15, h * w // 300))  # as many as the map holds
    ss = [make_scene(400 + i, persons, h=h, w=w) for i in range(2)]
    zero = np.zeros((2, 43, h, w), np.float32)
    return {"scenes": (np.stack([s["hms"] for s in ss]), np.stack([s["root_d"] for s in ss])),
            "noise": _noise(7, h, w), "zero": (zero, np.ones((2, h, w), np.float32)), "border": _border(h, w)}


@pytest.mark.parametrize("h,w", ASSOC_SIZES, ids=["%dx%d" % s for s in ASSOC_SIZES])
def test_association_on_the_scalar_nms_path_is_bit_exact(h, w):
    """extract (peaks, dense pair scores) and connect (both dist_flag modes, root_idx 0 and 2) against the oracle at map
    sizes where launch_nms takes nms_flag_kernel<false> (h*w % 128 != 0)."""
    from smap_b200.engine import Engine

    assert (h * w) % 128 != 0  # the condition launch_nms selects the scalar flag kernel on
    eng = Engine(0, max_batch=2, in_h=4 * h, in_w=4 * w)
    try:
        most = 0
        for name, (hms, rd) in assoc_inputs(h, w).items():
            hd, rdd = torch.from_numpy(hms).cuda(), torch.from_numpy(rd).cuda()
            peaks, scores = eng.extract(hd)
            torch.cuda.synchronize()
            peaks, scores = peaks.cpu().numpy(), scores.cpu().numpy()
            for i in range(2):
                rp, rs = assoc.extract(hms[i])
                assert np.array_equal(peaks[i], rp), "%s: peaks of frame %d" % (name, i)
                assert np.array_equal(scores[i], rs), "%s: pair scores of frame %d" % (name, i)
                most = max(most, int(rp[:, 0, 0].max()))
                if name == "border":  # no peak on the border; one peak, near its blob, 1-3 pixels inside
                    for f, side, d in BORDER_BLOBS:
                        c = d + (4 if side in ("left", "right") else 0)
                        if f == i:
                            assert int(rp[c, 0, 0]) == (1 if d else 0), (side, d, int(rp[c, 0, 0]))
            for root_idx in (0, 2):
                for dist_flag in (True, False):
                    bodies, counts = eng.connect(hd, rdd, root_idx, dist_flag)
                    torch.cuda.synchronize()
                    bodies, counts = bodies.cpu().numpy(), counts.cpu().numpy()
                    for i in range(2):
                        ob = assoc.connect(hms[i], rd[i], root_idx, dist_flag)
                        tag = "%s frame %d root_idx %d dist_flag %d" % (name, i, root_idx, dist_flag)
                        assert counts[i] == len(ob), tag
                        assert np.array_equal(bodies[i, :len(ob)], ob), tag
                        assert not bodies[i, len(ob):].any(), tag
        print("\n[assoc %dx%d] most peaks in one channel: %d" % (h, w, most))
        if h * w >= 4000:
            assert most == 127  # the noise frames reach the cap
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# whole path
# ---------------------------------------------------------------------------------------------------------------------
def test_whole_path_at_small_geometries_equals_the_oracle_chain():
    """infer_device records (do_flip off and on) at 32x32 B=2, 96x160 B=3 and 224x288 B=5 equal the oracle association
    and lift run on the backbone tensors of the same handle.  Across the geometries at least one frame has a person and
    one channel more than 20 peaks, so the comparison is not vacuous."""
    from smap_b200.engine import Engine, records_to_numpy, scale_row

    persons, most = 0, 0
    for H, W, B in [(32, 32, 2), (96, 160, 3), (224, 288, 5)]:
        eng = Engine(0, max_batch=B, in_h=H, in_w=W)
        try:
            eng.load_state_dict(schema.make_state_dict(0, "identity"))
            # uniform pixels plus 8x8-pixel blocks of Gaussian noise: channels with over 20 peaks on 56x72 maps
            g = torch.Generator().manual_seed(3)
            blocks = torch.kron(torch.randn(B, 3, H // 8, W // 8, generator=g), torch.ones(8, 8))
            x = (schema.make_input(B, H, W, seed=23) + blocks).cuda()
            sc = lift_numpy.default_scale(4 * W, 4 * H, net_w=W, net_h=H)
            scales = torch.from_numpy(np.stack([scale_row(sc)] * B)).cuda()
            hm, dd, rd = (t.clone() for t in eng.forward(x))
            hm_f = eng.forward(torch.flip(x, [-1]))[0].clone()
            for flip in (False, True):
                rec = records_to_numpy(eng.infer_device(x, scales, do_flip=flip))
                torch.cuda.synchronize()
                hms = smap_torch.rescale_reference_cuda(smap_torch.flip_merge(hm.clone(), hm_f) if flip else hm.clone())
                for i in range(B):
                    bodies, peaks, _ = assoc.connect(hms[i].cpu().numpy(), rd[i, 0].cpu().numpy(), return_all=True)
                    p2, p3, rdep = lift_numpy.lift(bodies, dd[i].cpu().numpy(), rd[i, 0].cpu().numpy(), sc)
                    n = int(rec["count"][i])
                    tag = "%dx%d frame %d flip %d" % (H, W, i, flip)
                    assert n == len(p2), tag
                    assert np.array_equal(rec["pred2d"][i, :n], p2), tag
                    assert np.array_equal(rec["root_depth"][i, :n], rdep), tag
                    np.testing.assert_allclose(rec["pred3d"][i, :n], p3, rtol=1e-12, atol=1e-12, err_msg=tag)
                    assert not rec["pred3d"][i, n:].any(), tag
                    persons += n
                    most = max(most, int(peaks[:, 0, 0].max()))
        finally:
            eng.close()
    print("\n[whole path] persons %d, most peaks in one channel %d" % (persons, most))
    assert persons > 0 and most > 20, (persons, most)


def test_two_handles_of_different_geometry_alternate_bit_exactly():
    """A 512x832 and a 32x32 handle in one process, calls alternating past the two eager runs (graph capture, replay):
    each returns what a handle of its geometry returned while no handle of the other geometry existed.  Process-wide
    state: the staged PAF kernel's shared-memory attribute (set per map size by assoc_configure), the once-per-process
    launch attributes and the tile table."""
    from smap_b200.engine import Engine, scale_row

    sd = schema.make_state_dict(0, "identity")
    geoms = {"512x832": (512, 832, 2), "32x32": (32, 32, 2)}
    args = {}
    for k, (H, W, B) in geoms.items():
        sc = lift_numpy.default_scale(4 * W, 4 * H, net_w=W, net_h=H)
        args[k] = (schema.make_input(B, H, W, seed=31).cuda(), torch.from_numpy(np.stack([scale_row(sc)] * B)).cuda())

    def handle(k):
        H, W, B = geoms[k]
        e = Engine(0, max_batch=B, in_h=H, in_w=W)
        e.load_state_dict(sd)
        return e

    def call(e, k):
        r = e.infer_device(*args[k]).cpu()
        torch.cuda.synchronize()
        return r

    alone = {}
    big = handle("512x832")
    alone["512x832"] = call(big, "512x832")
    big.close()
    small = handle("32x32")
    try:
        alone["32x32"] = call(small, "32x32")  # before any 512x832 handle exists again
        big = handle("512x832")
        try:
            for rnd in range(4):  # eager, eager, capture, replay
                for k, e in (("512x832", big), ("32x32", small)):
                    assert torch.equal(call(e, k), alone[k]), "%s, round %d" % (k, rnd)
        finally:
            big.close()
    finally:
        small.close()
