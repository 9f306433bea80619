"""GPU: every op of the real backbone plan, at its real geometry and tile choice, against a float64 reference of that one
layer fed the exact inputs the op consumed (the dumps of its producers, smapb_debug_dump), in bf16x3 and bf16.

An error in one edge tile, one 32-column epilogue chunk or one ring phase of one layer is diluted or hidden by the ReLUs
in the end-to-end bound of tests/test_backbone_gpu.py; here each op is compared on its own, element by element, by the
checker of tests/plan_check.py (check_ops; the bounds are given there).  For bf16x3, `-s` also prints the
per-channel max|y - r| / max|r_channel| (floored at 1e-3 max|r|) against the device-operand reference and against the
float64 layer computed from the unfolded state dict.  It is not asserted: channels that the ReLU or cancellation leave
small carry the error of their inputs' magnitude (up to a few 1e-3 at 832x512).
The checker is shown to flag deliberately wrong references, and forced tile widths are shown not to change a single bit
of any op, in bf16x3 and in bf16."""
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import _MUTATIONS, _X3_ONLY, _gid, check_switches, op_class, plan_summary  # noqa: E402

pytestmark = pytest.mark.gpu

BF16X3_GEOMS = [(64, 96, 2), (96, 160, 3), (512, 832, 8), (1024, 1024, 1)]
BF16_GEOMS = [(64, 96, 2), (96, 160, 3), (512, 832, 2)]
SWITCH_GEOMS = [(96, 160, 3), (512, 832, 8)]


@pytest.mark.parametrize("geom", BF16X3_GEOMS, ids=_gid)
def test_plan_ops_bf16x3(geom):
    s = plan_summary("bf16x3", geom)
    assert not s["failures"], "\n".join(s["failures"])


@pytest.mark.parametrize("geom", BF16_GEOMS, ids=_gid)
def test_plan_ops_bf16(geom):
    s = plan_summary("bf16", geom)
    assert not s["failures"], "\n".join(s["failures"])


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_checker_flags_wrong_references(precision):
    """The same comparison against deliberately wrong references (only host / reference-side tensors change)."""
    geoms = BF16X3_GEOMS if precision == "bf16x3" else BF16_GEOMS
    flagged = {}
    for g in geoms:
        for mut, f in plan_summary(precision, g)["flagged"].items():
            flagged.setdefault(mut, []).append(f)
    expect = set(_MUTATIONS) - (set(_X3_ONLY) if precision == "bf16" else set())
    assert set(flagged) == expect, "wrong references never tried: %s" % sorted(expect - set(flagged))
    assert all(len(fs) == len(geoms) for fs in flagged.values()), flagged  # every wrong reference on every geometry
    missed = [m for m, fs in flagged.items() if not all(fs)]
    assert not missed, "wrong references the checker accepted: %s" % missed


def test_plan_op_coverage():
    """Across the checked geometries every op kind of interest occurs, and no dumped op went unchecked."""
    seen, bns, up_tw, up_levels = set(), set(), set(), set()
    known = {"s2d", "stem_tc", "stem", "maxpool", "conv_f32", "conv"}
    for g in BF16X3_GEOMS:
        for op in plan_summary("bf16x3", g)["ops"]:
            assert op["kind"] in known, op  # check_ops fails on any kind it has no reference for
            cls = op_class(op)
            seen.add(cls)
            if "bn" in op:
                bns.add(int(op["bn"]))
            if cls == "up_residual":
                up_tw.add(int(op["tw"]))
                up_levels.add(re.search(r"\.up(\d)\.", op["name"]).group(1))
    for need in ("fused_pair_s1", "fused_pair_s2", "up_residual", "res_p1_p2", "head_f32", "tapexp", "stem_tc",
                 "maxpool", "s2d"):
        assert need in seen, "no %s op checked (seen: %s)" % (need, sorted(seen))
    assert up_levels == {"2", "3", "4"}, up_levels
    assert {32, 64, 128} <= bns, bns
    assert len(up_tw) >= 2, up_tw


@pytest.mark.parametrize("geom", SWITCH_GEOMS, ids=_gid)
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_forced_tile_widths_keep_the_bits(precision, geom, monkeypatch):
    """Every forced tile width gives every op the same bits as the default plan.  (Switches held in function-local
    statics, SMAPB_NO_GRAPH / SMAPB_DEBUG_STOP, cannot be toggled in one process.)"""
    check_switches(geom, monkeypatch, precision)
