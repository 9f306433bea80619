"""GPU: fp16's range guard.  In the fp16 precision every kernel that stores an fp16 activation it computed (the conv epilogue
in all its variants, the CUDA-core stem, s2d) must store exactly +-65504 for a value beyond the range, never
inf or NaN, and add one to the handle's saturation counter per clamped element - the counter is the only sign a user gets
that the outputs are not the model's.

The reference is the float64 one of tests/plan_check.py (the value before the store, r) with its accumulation bound b,
and the store's clamp on top: check_ops in fp16.  Elements split three ways:
  * sure-over, |r| - b > 65504: the output is exactly sign(r) 65504 and the element is counted;
  * sure-in, |r| + b <= 65504: not counted, |y - r| <= 1/2 ulp_fp16(y) + b as before;
  * band, the rest: either outcome, |y - clamp(r)| <= 1/2 ulp_fp16(y) + b.
A forward's device count must lie in [sum sure-over, sum sure-over + sum band] over every fp16-storing op, and the state
dicts keep the band smaller than the sure-over count of every op class that saturates, so a class whose clamps go
uncounted (or a count of rows outside the output) fails.

  * whole plans (default, and the CUDA-core stem fallback) at 96x64 B2, 288x224 B5 (odd levels: partial tiles
    both ways) and 32x32 B2 (1x1 deepest level, flat M = 2), with state dicts that drive chosen units over the range
    through their BN bias (positive, and negative on a unit without a ReLU) and keep the saturated channels from
    spreading: consumers' weights on them are zeroed, residual consumers' biases send them below the ReLU;
  * the first forward of a fresh handle counts that forward and nothing of the plan build's autotuning launches;
  * single convolutions through conv_test at every tile width, flat and tiled partial tiles, residuals, negative biases,
    post-ReLU skips at -65504, one saturating lane per warp and whole saturating chunks: exact counts, no band;
  * counter semantics: eager, graph capture and replay, flip, two handles, reset; bf16x3 and bf16 count nothing on the same
    weights and pass their per-op checks; s2d's mapping of NaN / inf / out-of-range pixels.
(-s prints, per plan, the sure-over count per op class, the band, the device count and the worst |y - clamp(r)| / bound.)"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import lift_numpy, smap_torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import (FP16_MAX, ROLES, SEED, _acc_bound, _consumers, _gid, _nchw, _nhwc, check_ops,  # noqa: E402
                        check_plan, clamp_check, no_tf32, op_class, plan_ops, split3)

pytestmark = pytest.mark.gpu

S = 1.7e5  # BN bias of a saturated channel: ~1e5 beyond the range, so the accumulation bound never reaches the limit
GEOMS = [(64, 96, 2), (224, 288, 5), (32, 32, 2)]
PLANS = {
    "default": ({}, ("conv1x1", "conv3x3", "residual", "fused_pair_s1", "fused_pair_s2", "up_residual", "res_p1_p2",
                     "stem_tc")),
    "cuda_stem": ({"SMAPB_STEM": "cuda"}, ("conv3x3", "residual", "fused_pair_s2", "res_p1_p2", "stem")),
}


# ---------------------------------------------------------------------------------------------------------------------
# the interval of the device count
# ---------------------------------------------------------------------------------------------------------------------
def report(tag, s, n):
    print("\n[fp16 saturation %s] device count %d in [%d, %d]: band %d, negative sure-over %d" % (tag, n, s["lo"], s["hi"],
                                                                                             s["band"], s["neg"]))
    for cls in sorted(set(s["over"]) | set(s["worst"])):
        print("  %-14s sure-over %8d   worst |y - clamp(r)| / bound %.3g" % (cls, s["over"].get(cls, 0),
                                                                           s["worst"].get(cls, 0.0)))


def assert_interval(s, n):
    assert not s["failures"], "\n".join(s["failures"])
    assert s["lo"] <= n <= s["hi"], "device count %d outside [%d, %d]" % (n, s["lo"], s["hi"])
    # a class that counted nothing, or dropped more of its clamps than the band allows, moves n out of the interval
    for cls, k in s["over"].items():
        assert s["band"] < k, "band %d not below the sure-over count %d of %s" % (s["band"], k, cls)


# ---------------------------------------------------------------------------------------------------------------------
# saturating state dicts
# ---------------------------------------------------------------------------------------------------------------------
_GRAPHS = {}


def op_graph(H, W, B):
    """The plan's op descriptions under the current environment (they do not depend on the weights)."""
    from smap_b200.engine import Engine

    key = (H, W, B, os.environ.get("SMAPB_STEM"))
    if key not in _GRAPHS:
        eng = Engine(0, max_batch=B, in_h=H, in_w=W)
        try:
            eng.load_state_dict(smap_torch.make_state_dict(SEED, "random"), "fp16")
            _GRAPHS[key] = plan_ops(eng, B)[1]
        finally:
            eng.close()
    return _GRAPHS[key]


def _unit_of(op, role):
    """The state-dict unit whose weights multiply input `role` of conv op `op`."""
    if "in2" in op:
        base = op["name"][:-len("fused_conv3_downsample")]
        return base + ("downsample" if role == "in2" else "conv_bn_relu3")
    return op["name"]


def _containable(ops, uses, i, sign):
    """Whether every consumer of op i can be kept from carrying a saturated channel of sign `sign` further."""
    for j in uses.get(i, []):
        c = ops[j]
        for role in [r for r in ROLES if c.get(r) == str(i)]:
            if c["kind"] == "maxpool":
                if not _containable(ops, uses, j, sign):
                    return False
            elif c["kind"] == "conv_f32" or (c["kind"] == "conv" and role in ("in", "in2")):
                continue
            elif c["kind"] == "conv" and role in ("res", "up") and int(c["relu"]) and "p1" not in c:
                continue
            else:
                return False
    return True


def _contain(sd, ops, uses, i, cs, sign):
    """Zero the consumers' weights on channels cs of op i's output, or (residual / up inputs) push the consumer's channels
    below its ReLU.  fp32 heads keep their +-65504 inputs."""
    for j in uses.get(i, []):
        c = ops[j]
        for role in [r for r in ROLES if c.get(r) == str(i)]:
            if c["kind"] == "maxpool":
                _contain(sd, ops, uses, j, cs, sign)
            elif c["kind"] == "conv" and role in ("in", "in2"):
                sd[_unit_of(c, role) + ".conv.weight"][:, cs] = 0.0
            elif c["kind"] == "conv" and role in ("res", "up") and sign > 0:
                sd[c["name"] + ".bn.bias"][cs] = -S


def _units_of_target(ops, op):
    if op["kind"] in ("stem_tc", "stem"):
        return ["top.conv"]
    return [_unit_of(op, "in")]


def saturating_state_dict(ops, plan):
    """make_state_dict(SEED, "random") with one unit of every op class of PLANS[plan] driven over the range on two
    channels (one per 32-channel chunk), plus, on the default plan, an up_conv (no ReLU) driven below -65504."""
    sd = {k: v.clone() for k, v in smap_torch.make_state_dict(SEED, "random").items()}
    uses = _consumers(ops)
    size = lambda o: np.prod([int(v) for v in o["out"].split("x")[:3]])  # noqa: E731
    targets = []
    for cls in PLANS[plan][1]:
        cand = [o for o in ops if op_class(o) == cls and (o["kind"] != "conv" or int(o["relu"]))
                and _containable(ops, uses, o["idx"], 1)]
        assert cand, "no containable %s op" % cls
        targets.append((max(cand, key=size), 1))  # the largest output: most elements per saturated channel
    if plan == "default":
        cand = [o for o in ops if op_class(o) == "conv1x1" and not int(o["relu"]) and _containable(ops, uses, o["idx"], -1)]
        assert cand, "no conv without a ReLU"
        targets.append((max(cand, key=size), -1))
    for k, (op, sign) in enumerate(targets):
        cs = [(5 + 13 * k) % 64, (37 + 13 * k) % 64]
        for unit in _units_of_target(ops, op):
            sd[unit + ".bn.bias"][cs] = sign * S
        _contain(sd, ops, uses, op["idx"], cs, sign)
    return sd, [("+".join(_units_of_target(ops, op)), sign) for op, sign in targets]


def _images(B, H, W):
    return smap_torch.make_input(B, H, W, seed=SEED + 1).cuda(), smap_torch.make_input(B, H, W, seed=SEED + 2).cuda()


# ---------------------------------------------------------------------------------------------------------------------
# 1-2: every fp16-storing op of whole plans
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: _gid(g, width_first=True))
def test_plan_saturation_is_clamped_and_counted(geom, plan, monkeypatch):
    from smap_b200.engine import Engine

    no_tf32()
    H, W, B = geom
    for k, v in PLANS[plan][0].items():
        monkeypatch.setenv(k, v)  # read at plan build
    ops = op_graph(H, W, B)
    sd, targets = saturating_state_dict(ops, plan)
    warm, img = _images(B, H, W)
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, "fp16")
        eng.forward(warm)
        eng.saturation_count(reset=True)
        outs = eng.forward(img)
        n = eng.saturation_count()
        s = check_ops(eng, B, sd, img, outs, "fp16")
        for o in outs:
            assert torch.isfinite(o).all()
    finally:
        eng.close()
    torch.cuda.empty_cache()
    report("%s %s" % (plan, _gid(geom, width_first=True)), s, n)
    print("  targets: %s" % ", ".join("%s%s" % ("-" if sg < 0 else "+", t) for t, sg in targets))
    assert_interval(s, n)
    for cls in PLANS[plan][1]:
        assert s["over"].get(cls, 0) > 0, "no sure-over element in %s (%s)" % (cls, sorted(s["over"]))
    if plan == "default":
        assert s["neg"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# 3: a fresh handle's first forward counts that forward only
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("autotune", [True, False], ids=["autotune", "no_autotune"])
def test_first_forward_of_a_fresh_handle_counts_one_forward(autotune, monkeypatch):
    """The plan is built by the first forward; with autotuning its trial launches run every conv on zeroed activations
    (output = bias) and must not add to the user's counter.  The process-wide tile table is made to hold no valid fp16
    row (rows are given a width no kernel has, which the autotuner measures again), so the plan build autotunes - or,
    with SMAPB_NO_AUTOTUNE, takes the cost model - whatever ran before."""
    from smap_b200 import _lib
    from smap_b200.engine import Engine, get_tile_table

    no_tf32()
    H, W, B = GEOMS[0]
    sd, _ = saturating_state_dict(op_graph(H, W, B), "default")
    _, img = _images(B, H, W)
    lib = _lib.load()
    table = get_tile_table()

    def stale():  # fp16 rows holding the invalid width
        return sum(1 for r in (line.split("\t") for line in get_tile_table().splitlines())
                   if r[0].endswith(" f16") and r[1] == "96")

    rows = [line.split("\t") for line in table.splitlines()]
    lib.smapb_set_tile_table("".join("%s\t96\t1\n" % r[0] for r in rows if r[0].endswith(" f16")).encode())
    n_stale = stale()
    eng = None
    try:
        if not autotune:
            monkeypatch.setenv("SMAPB_NO_AUTOTUNE", "1")  # read at handle creation
        eng = Engine(0, max_batch=B, in_h=H, in_w=W)
        eng.load_state_dict(sd, "fp16")
        outs = eng.forward(img)
        n = eng.saturation_count()
        s = check_ops(eng, B, sd, img, outs, "fp16")
        tuned = n_stale - stale()
    finally:
        if eng is not None:
            eng.close()
        lib.smapb_set_tile_table(table.encode())
    report("fresh handle %s %s" % ("autotune" if autotune else "SMAPB_NO_AUTOTUNE", _gid(GEOMS[0], width_first=True)), s, n)
    print("  fp16 tile-table rows re-measured by this plan build: %d" % tuned)
    if autotune:
        assert tuned > 0, "the plan build did not autotune"
    else:
        assert tuned == 0
    assert_interval(s, n)


# ---------------------------------------------------------------------------------------------------------------------
# 4: single convolutions, exact counts
# ---------------------------------------------------------------------------------------------------------------------
_KCASES = {  # B, H, W, Cin, Cout, k, stride, relu, epilogue inputs
    "tiled3x3_res": (2, 16, 24, 64, 128, 3, 1, True, "res"),
    "tiled3x3_posts": (2, 16, 24, 64, 128, 3, 1, True, "posts"),
    "flat1x1_m126": (2, 7, 9, 64, 128, 1, 1, False, ""),
    "flat1x1_m126_res": (2, 7, 9, 64, 128, 1, 1, True, "res"),
    "partial3x3": (2, 13, 19, 64, 128, 3, 1, False, ""),
    "partial3x3_s2": (2, 13, 19, 64, 128, 3, 2, True, "res"),
    "partial1x1_s2_posts": (2, 13, 19, 128, 128, 1, 2, True, "posts"),
}


def _kernel_operands(name):
    """fp16-representable operands (conv_test converts them without a clamp).  Channels 32-63 (one whole 32-column
    chunk) get +1e5 biases, channels 5 and 9 +1e5 and -1e5; a residual adds 65504 at one element of channel 17 over a
    +1000 bias (one saturating lane in its warp); posts put -65504 + -65504 on all of channel 20 after the ReLU."""
    B, H, W, Cin, Cout, k, stride, relu, extra = _KCASES[name]
    g = torch.Generator(device="cpu").manual_seed(17)
    h = lambda t: t.half().float().cuda()  # noqa: E731
    x = h(torch.randn(B, H, W, Cin, generator=g))
    w = h(torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5)
    b = torch.randn(Cout, generator=g) * 0.1
    b[32:64] = 1.0e5
    b[5], b[9] = 1.0e5, -1.0e5
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    res = post1 = post2 = None
    if extra == "res":
        b[17] = 1000.0
        rr = torch.randn(B, Ho, Wo, Cout, generator=g)
        rr[B - 1, Ho - 1, Wo // 2, 17] = FP16_MAX
        res = h(rr)
    if extra == "posts":
        p1, p2 = torch.rand(B, Ho, Wo, Cout, generator=g), torch.rand(B, Ho, Wo, Cout, generator=g)
        p1[..., 20] = -FP16_MAX
        p2[..., 20] = -FP16_MAX
        post1, post2 = h(p1), h(p2)
    return x, w, b.cuda(), res, post1, post2


def _kernel_reference(name, x, w, b, res, post1, post2):
    """-> (r, pre, q) in fp64, q^2 the sum of the squared terms of each element."""
    B, H, W, Cin, Cout, k, stride, relu, _ = _KCASES[name]
    conv = lambda xx, ww: _nhwc(F.conv2d(_nchw(xx), ww, stride=stride, padding=k // 2))  # noqa: E731
    pre = conv(x.double(), w.double()) + b.double()
    sq = conv(x.double() ** 2, w.double() ** 2) + b.double() ** 2
    if res is not None:
        pre, sq = pre + res.double(), sq + res.double() ** 2
    r = F.relu(pre) if relu else pre
    for p in (post1, post2):
        if p is not None:
            r, sq = r + p.double(), sq + p.double() ** 2
    return r, pre, sq.sqrt()


@pytest.mark.parametrize("name", list(_KCASES))
def test_conv_saturation_count_is_exact_at_every_tile_width(eng16, name, monkeypatch):
    B, H, W, Cin, Cout, k, stride, relu, _ = _KCASES[name]
    x, w, b, res, post1, post2 = _kernel_operands(name)
    r, pre, q = _kernel_reference(name, x, w, b, res, post1, post2)
    op = {"kind": "conv", "k": "%dx%d" % (k, k), "cin": str(Cin)}
    bnd = _acc_bound(op, q, r, pre)
    over, _, band = split3(r, bnd)
    assert not band.any(), "operands leave %d elements in the band" % int(band.sum().item())
    n_over = int(over.sum().item())
    assert over[..., 32:64].all() and over[..., 5].all()
    if not relu:
        assert (over & (r < 0))[..., 9].all()
    if res is not None:
        assert int(over[..., 17].sum().item()) == 1  # one element: one lane of its warp
    if post1 is not None:
        assert (over & (r < 0))[..., 20].all()
    first = None
    eng16.saturation_count(reset=True)
    for tile in ("128", "64", "32"):
        monkeypatch.setenv("SMAPB_FORCE_TILE", tile)
        y = eng16.conv_test(x, w, b, res=res, stride=stride, relu=relu, precision="fp16", post1=post1, post2=post2)
        n = eng16.saturation_count(reset=True)
        y = y.double()
        assert torch.isfinite(y).all()
        _, _, err, bad = clamp_check(y, r, bnd)
        assert not bad, "tile %s: %s" % (tile, "; ".join(bad))
        if relu and post1 is None:
            assert (y[pre < -bnd] == 0).all()
        assert n == n_over, "tile %s: count %d, %d elements beyond the range" % (tile, n, n_over)
        if first is None:
            first = y
            print("\n[fp16 conv_test %s] %d of %d elements clamped, worst |y - clamp(r)| / bound %.3g"
                  % (name, n_over, r.numel(), err))
        assert torch.equal(y, first), "tile %s changes the bits" % tile


def test_conv_test_timing_and_timeline_launches_do_not_count(eng16, monkeypatch):
    """conv_test's timed repetitions and its SMAPB_TIMELINE launch re-run the conv: only the result launch counts."""
    x, w, b, res, _, _ = _kernel_operands("tiled3x3_res")
    eng16.saturation_count(reset=True)
    eng16.conv_test(x, w, b, res=res, precision="fp16")
    n = eng16.saturation_count(reset=True)
    assert n > 0
    eng16.conv_test(x, w, b, res=res, precision="fp16", time_it=True)
    assert eng16.saturation_count(reset=True) == n
    monkeypatch.setenv("SMAPB_TIMELINE", "1")
    eng16.conv_test(x, w, b, res=res, precision="fp16")
    assert eng16.saturation_count(reset=True) == n


@pytest.fixture(scope="module")
def eng16():
    from smap_b200.engine import Engine

    no_tf32()
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: counter semantics on the whole path
# ---------------------------------------------------------------------------------------------------------------------
def _scales(B, H, W):
    from smap_b200.engine import scale_row

    sc = lift_numpy.default_scale(4 * W, 4 * H, net_w=W, net_h=H)
    return torch.from_numpy(np.stack([scale_row(sc)] * B)).cuda()


def test_every_forward_counts_once_eager_graph_and_flip():
    from smap_b200.engine import Engine

    H, W, B = GEOMS[0]
    sd, _ = saturating_state_dict(op_graph(H, W, B), "default")
    _, x = _images(B, H, W)
    xf = torch.flip(x, dims=[3])
    scales = _scales(B, H, W)
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, "fp16")
        eng.forward(x)
        eng.saturation_count(reset=True)
        eng.forward(x)
        c = eng.saturation_count(reset=True)
        eng.forward(xf)
        cf = eng.saturation_count(reset=True)
        assert c > 0 and cf > 0
        seen = []
        for i in range(4):  # 2 eager runs, then graph capture and replay
            eng.infer_device(x, scales)
            seen.append(eng.saturation_count())
        assert seen == [c * (i + 1) for i in range(4)], (c, seen)
        eng.saturation_count(reset=True)
        seen = []
        for i in range(4):
            eng.infer_device(x, scales, do_flip=True)
            seen.append(eng.saturation_count())
        assert seen == [(c + cf) * (i + 1) for i in range(4)], (c, cf, seen)
        print("\n[fp16 saturation counter] one forward %d, flipped %d, infer_device x4 and flip x4 counted each" % (c, cf))
    finally:
        eng.close()


def test_handles_count_independently_and_reset():
    from smap_b200.engine import Engine

    H, W, B = GEOMS[0]
    sd, _ = saturating_state_dict(op_graph(H, W, B), "default")
    _, x = _images(B, H, W)
    e1 = Engine(0, max_batch=B, in_h=H, in_w=W)
    e2 = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        e1.load_state_dict(sd, "fp16")
        e2.load_state_dict(sd, "fp16")
        e1.forward(x)
        c = e1.saturation_count()
        assert c > 0 and e2.saturation_count() == 0
        e2.forward(x)
        e2.forward(x)
        assert e1.saturation_count() == c and e2.saturation_count() == 2 * c
        assert e1.saturation_count(reset=True) == c
        assert e1.saturation_count() == 0 and e2.saturation_count() == 2 * c
    finally:
        e1.close()
        e2.close()


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_bf16_precisions_hold_the_range_and_count_nothing(precision):
    from smap_b200.engine import Engine

    H, W, B = GEOMS[0]
    sd, _ = saturating_state_dict(op_graph(H, W, B), "default")
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, precision)
        s = check_plan(precision, H, W, B, eng=eng, sd=sd)
        assert eng.saturation_count() == 0
        ys = [eng.forward(img) for img in _images(B, H, W)]
        torch.cuda.synchronize()
        assert all(torch.isfinite(o).all() for y in ys for o in y)
        assert eng.saturation_count() == 0
    finally:
        eng.close()
    assert not s["failures"], "\n".join(s["failures"])


_SPECIAL = [float("nan"), float("inf"), -float("inf"), 1.0e5, -1.0e5, FP16_MAX, -FP16_MAX, 65505.0, -65505.0, 65519.0]


def test_s2d_maps_non_finite_and_out_of_range_pixels():
    """NaN -> -65504 and beyond the range -> +-65504 (common.cuh ElemF16::clamp), each counted; the pixels are 16 apart,
    so no 7x7 stem window sees two of them and nothing downstream saturates."""
    from smap_b200.engine import Engine

    no_tf32()
    H, W, B = GEOMS[0]
    sd = smap_torch.make_state_dict(SEED, "random")
    warm, img = _images(B, H, W)
    for i, v in enumerate(_SPECIAL):
        img[i % B, i % 3, 8 + 16 * (i // 5), 8 + 16 * (i % 5)] = v
    n_out = sum(1 for v in _SPECIAL if not abs(v) <= FP16_MAX)
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, "fp16")
        eng.forward(warm)
        eng.saturation_count(reset=True)
        outs = eng.forward(img)
        n = eng.saturation_count()
        s = check_ops(eng, B, sd, img, outs, "fp16")
        for o in outs:
            assert torch.isfinite(o).all()
    finally:
        eng.close()
    report("special pixels %s" % _gid(GEOMS[0], width_first=True), s, n)
    assert s["over"] == {"s2d": n_out}, s["over"]
    assert s["band"] == 0
    assert n == n_out
    assert not s["failures"], "\n".join(s["failures"])
