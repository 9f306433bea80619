"""GPU: the fp16 precision (SMAPB_PREC_FP16): fp16 operands and activations, fp32 accumulation, stores clamped to +-65504.

  * single convolutions (the CASES of tests/plan_check.py) against a float64 reference built from the fp16-rounded
    operands the device holds, by the conv-level checker check_conv (tests/plan_check.py): |y - r| <= 1/2 ulp_fp16(y) +
    _acc_bound, and the same checker flags a reference built from bf16-rounded operands (every kernel instance and
    epilogue form at the edges of the tiling: tests/test_conv_edges_gpu.py);
  * saturation: outputs beyond +-65504 are exactly +-65504, never inf / NaN, and counted; folded weights beyond the range
    are rejected by finalize;
  * every op of the real plan against a float64 reference of its own layer, by the checker of tests/plan_check.py that
    tests/test_plan_ops_gpu.py runs for bf16x3 and bf16 (wrong references flagged, heads checked), and forced tile
    widths that must not change a bit;
  * the whole backbone against the fp32 oracle next to bf16 and cuDNN with TF32 (the reference's own GPU numerics);
  * the whole path (records) on bench.py's first batch next to bf16x3.

Measured on one H100 80GB HBM3 (400 W power limit), max|a - b| / max|ref| against the fp32 oracle:

    geometry              tensor   fp16      bf16      cuDNN TF32
    832x512 B2 identity   hm2d     1.52e-3   1.09e-2   1.57e-3
                          detd     3.13e-3   2.57e-2   3.10e-3
                          rootd    4.74e-3   3.35e-2   4.70e-3
    832x512 B2 random     hm2d     6.15e-4   4.38e-3   4.05e-4
                          detd     4.73e-4   3.22e-3   3.86e-4
                          rootd    8.72e-4   8.33e-3   9.23e-4
    1024x1024 B1 identity hm2d     1.69e-3   1.17e-2   1.87e-3
                          detd     3.16e-3   2.19e-2   3.10e-3
                          rootd    4.99e-3   3.64e-2   4.56e-3

fp16 lands where the reference's own cuDNN-TF32 run lands, 7x below bf16.

(-s prints the table; FP16_BOUND keeps a factor >= 2 over the worst fp16 value.)"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import smap_torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import (CASES, FP16_MAX, _TILE_CASES, _K, _gid, _nchw, _nhwc, assert_checked, check_conv,  # noqa: E402
                        check_switches, conv_inputs, legacy_op, no_tf32, op_class, plan_summary, run_conv)

pytestmark = pytest.mark.gpu

FP16_BOUND = 1e-2  # backbone vs fp32 oracle, max|a - b| / max|ref| per tensor (measured <= 4.99e-3, see above)


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    no_tf32()
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


@pytest.mark.parametrize("case", CASES)
def test_conv_fp16_matches_fp64_of_device_operands(eng, case):
    op = legacy_op(case)
    t = conv_inputs(op, hash(case) % (2 ** 31))
    y = run_conv(eng, op, t, "fp16")
    torch.cuda.synchronize()
    assert torch.equal(y, y.half().float()), "outputs are not fp16 values"
    j = check_conv(op, y, t, "fp16")
    assert not j["bad"], "\n".join(j["bad"])
    assert not j["over"].any() and not j["band"].any()
    assert eng.saturation_count(reset=True) == 0


def test_checker_flags_a_bf16_operand_reference(eng):
    """On the largest-K case the checker that passes fp16 rejects a reference built from bf16-rounded operands: the bound
    resolves fp16's 4x finer operand rounding."""
    case = max(CASES, key=lambda c: c[3] * c[5] * c[5])
    op = legacy_op(case)
    t = conv_inputs(op, hash(case) % (2 ** 31))
    y = run_conv(eng, op, t, "fp16")
    torch.cuda.synchronize()
    right, wrong = check_conv(op, y, t, "fp16"), check_conv(op, y, t, "fp16", operands="bf16")
    print("\n[fp16 checker] K=%d: fp16-operand reference %.3g, bf16-operand reference %.3g of the elements outside the"
          " bound" % (_K(op), right["share"], wrong["share"]))
    assert not right["bad"], right["bad"]
    assert wrong["share"] > 0.05


@pytest.mark.parametrize("case", _TILE_CASES)
def test_fp16_every_tile_width_and_every_run_gives_the_same_bits(eng, monkeypatch, case):
    op = legacy_op(case)
    t = conv_inputs(op, 11)
    first, n = None, 0
    for tile in ("128", "64", "32"):
        if int(op["cout"]) % int(tile):
            continue
        monkeypatch.setenv("SMAPB_FORCE_TILE", tile)
        for _ in range(2):
            y = run_conv(eng, op, t, "fp16")
            torch.cuda.synchronize()
            if first is None:
                first = y
                j = check_conv(op, y, t, "fp16")
                assert not j["bad"], "\n".join(j["bad"])
            assert torch.equal(y, first), "tile %s: %d elements differ" % (tile, (y != first).sum().item())
        n += 1
    assert n >= 2


# ---------------------------------------------------------------------------------------------------------------------
# saturation
# ---------------------------------------------------------------------------------------------------------------------
def _saturating_conv():
    g = torch.Generator(device="cpu").manual_seed(3)
    B, H, W, C = 2, 16, 24, 64
    x = torch.randn(B, H, W, C, generator=g).cuda()
    w = (torch.randn(C, C, 3, 3, generator=g) / (9 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    b[0], b[5], b[33] = 7.0e4, -7.0e4, FP16_MAX
    w[33] *= 1000.0  # channel 33 spreads +-1000s around 65504: its pixels go either way
    return x, w, b


def test_saturation_clamps_counts_and_resets(eng):
    x, w, b = _saturating_conv()
    eng.saturation_count(reset=True)
    y = eng.conv_test(x, w, b, relu=False, precision="fp16").double()
    r = _nhwc(F.conv2d(_nchw(x.half().double()), w.half().double(), padding=1)) + b.double()
    over = r.abs() > FP16_MAX
    margin = (r.abs() - FP16_MAX).abs() < 0.01  # too close to the limit for the fp32 accumulation to decide
    assert not margin.any()
    assert torch.isfinite(y).all()
    assert torch.equal(y[over], torch.sign(r[over]) * FP16_MAX)
    assert (y[~over].abs() <= FP16_MAX).all()
    n = int(over.sum().item())
    assert over[..., 0].all() and over[..., 5].all() and 0 < over[..., 33].sum() < over[..., 33].numel()
    assert eng.saturation_count() == n
    assert eng.saturation_count(reset=True) == n
    assert eng.saturation_count() == 0
    # the same conv in bf16x3 holds the values and never touches the counter
    y3 = eng.conv_test(x, w, b, relu=False, precision="bf16x3").double()
    assert (y3[..., 0] > FP16_MAX).all() and (y3[..., 5] < -FP16_MAX).all()
    assert eng.saturation_count() == 0


def test_finalize_rejects_weights_beyond_the_fp16_range():
    from smap_b200.engine import Engine, SmapB200Error

    x = smap_torch.make_input(1, 64, 96, seed=1).cuda()
    e = Engine(0, max_batch=1, in_h=64, in_w=96)
    try:
        # a unit the plan runs on its own, and one it runs only inside a fused conv3 + downsample pair: the error names
        # the state-dict unit either way
        for unit in ("stage1.downsample.layer2.1.conv_bn_relu2", "stage0.downsample.layer3.0.downsample"):
            sd = dict(smap_torch.make_state_dict(0, "identity"))
            sd[unit + ".conv.weight"] = sd[unit + ".conv.weight"].clone()
            sd[unit + ".conv.weight"][3, 1, 0, 0] = 1.0e5
            with pytest.raises(SmapB200Error, match=unit.replace(".", r"\.") + " exceeds"):
                e.load_state_dict(sd, "fp16")
            with pytest.raises(SmapB200Error, match="not finalized"):
                e.forward(x)
        e.load_state_dict(sd, "bf16x3")  # bf16 keeps fp32's range
        e.forward(x)
        torch.cuda.synchronize()
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# per-op parity of the real plan
# ---------------------------------------------------------------------------------------------------------------------
PLAN_GEOMS = [(64, 96, 2), (512, 832, 2), (1024, 1024, 1)]


@pytest.mark.parametrize("geom", PLAN_GEOMS, ids=_gid)
def test_plan_ops_fp16(geom):
    s = plan_summary("fp16", geom)
    assert_checked(s, "fp16")
    seen = {op_class(o) for o in s["ops"]}
    for need in ("conv1x1", "conv3x3", "residual", "fused_pair_s1", "fused_pair_s2", "up_residual", "res_p1_p2", "head_f32",
                 "tapexp", "stem_tc", "maxpool", "s2d"):
        assert need in seen, "no %s op checked (seen: %s)" % (need, sorted(seen))


@pytest.mark.parametrize("geom", [(64, 96, 2), (512, 832, 2)], ids=_gid)
def test_fp16_forced_tile_widths_keep_the_bits(geom, monkeypatch):
    from smap_b200.engine import get_tile_table

    check_switches(geom, monkeypatch, "fp16")
    assert any(line.split("\t")[0].endswith(" f16") for line in get_tile_table().splitlines())  # fp16 rows of their own


# ---------------------------------------------------------------------------------------------------------------------
# whole backbone, whole path
# ---------------------------------------------------------------------------------------------------------------------
def rel(a, b):
    return (a - b).abs().max().item() / b.abs().max().item()


@pytest.mark.parametrize("H,W,B,bn", [(512, 832, 2, "identity"), (512, 832, 2, "random"), (1024, 1024, 1, "identity")],
                         ids=["832x512_b2_identity", "832x512_b2_random", "1024x1024_b1_identity"])
def test_backbone_fp16_vs_fp32_oracle(H, W, B, bn, capsys):
    from smap_b200.engine import Engine

    sd = smap_torch.make_state_dict(0, bn)
    x = smap_torch.make_input(B, H, W, seed=1).cuda()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    no_tf32()
    ref = smap_torch.smap_forward(sd_dev, x)
    torch.backends.cudnn.allow_tf32 = True  # PyTorch's default: the reference's own SMAP.cuda() convolutions
    tf32 = smap_torch.smap_forward(sd_dev, x)
    no_tf32()
    errs = {"tf32": [rel(a, b) for a, b in zip(tf32, ref)]}
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        for prec in ("bf16", "fp16"):
            eng.load_state_dict(sd, prec)
            out = eng.forward(x)
            torch.cuda.synchronize()
            for a in out:
                assert torch.isfinite(a).all()
            errs[prec] = [rel(a, b) for a, b in zip(out, ref)]
        assert eng.saturation_count() == 0
        # fp16 (still loaded): one image alone gives the bits it has within its batch
        o1 = eng.forward(x[B - 1:B])
        torch.cuda.synchronize()
        for a, b in zip(o1, out):
            assert torch.equal(a[0], b[B - 1])
    finally:
        eng.close()
    with capsys.disabled():
        print("\n[fp16 backbone %dx%d B=%d %s] max|a-b|/max|ref| vs the fp32 oracle" % (W, H, B, bn))
        for i, name in enumerate(("hm2d", "detd", "rootd")):
            print("  %-6s fp16 %.2e  bf16 %.2e  cuDNN-TF32 %.2e" % (name, errs["fp16"][i], errs["bf16"][i], errs["tf32"][i]))
    for i, name in enumerate(("hm2d", "detd", "rootd")):
        assert errs["fp16"][i] < errs["bf16"][i], name
        assert errs["fp16"][i] < FP16_BOUND, (name, errs["fp16"][i])


def _peak_set(peaks):
    out = set()
    for c in range(peaks.shape[0]):
        for k in range(1, int(peaks[c, 0, 0]) + 1):
            out.add((c, int(round(float(peaks[c, k, 0]) * 8)), int(round(float(peaks[c, k, 1]) * 8))))
    return out


def test_whole_path_fp16_on_the_bench_batch(capsys):
    """infer_device in fp16 on bench.py's first batch (8 x 832x512): finite records, graph replay == eager, no
    saturation; person and candidate agreement with bf16x3 are printed (noise-like random-init maps: a candidate within
    the backbone's error of the 0.2 threshold or of a neighbour flips, as in tests/test_e2e_chain_gpu.py)."""
    from oracle import lift_numpy
    from smap_b200 import schema
    from smap_b200.engine import Engine, records_to_numpy, scale_row

    no_tf32()
    B, H, W = 8, 512, 832
    sd = schema.make_state_dict(0, "identity")
    x = schema.make_input(B, H, W, seed=1).cuda()
    scales = torch.from_numpy(np.stack([scale_row(lift_numpy.default_scale(1920, 1080))] * B)).cuda()
    res = {}
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        for prec in ("bf16x3", "fp16"):
            eng.load_state_dict(sd, prec)
            runs = [eng.infer_device(x, scales).clone() for _ in range(4)]  # 2 eager, then graph capture and replay
            torch.cuda.synchronize()
            for r in runs[1:]:
                assert torch.equal(r, runs[0]), prec
            hm = eng.merge_scale(eng.forward(x)[0], None, True)
            peaks, _ = eng.extract(hm)
            torch.cuda.synchronize()
            res[prec] = (records_to_numpy(runs[0]), peaks.cpu().numpy())
        assert eng.saturation_count() == 0
    finally:
        eng.close()
    r16, p16 = res["fp16"]
    r3, p3 = res["bf16x3"]
    for f in ("pred3d", "root_depth", "pred2d"):
        assert np.isfinite(r16[f]).all(), f
    tot = flips = persons = matched = 0
    for i in range(B):
        s16, s3 = _peak_set(p16[i]), _peak_set(p3[i])
        tot += len(s16 | s3)
        flips += len(s16 ^ s3)
        n3, n16 = int(r3["count"][i]), int(r16["count"][i])
        persons += n3
        for k in range(n3):
            a = r3["pred2d"][i, k]
            for j in range(n16):
                b = r16["pred2d"][i, j]
                if ((a[:, 3] != 0) == (b[:, 3] != 0)).all() and np.abs(a[:, :2] - b[:, :2]).max() < 0.05:
                    matched += 1
                    break
    with capsys.disabled():
        print("\n[fp16 whole path] frames=%d persons bf16x3=%d fp16=%d, fp16 persons matching a bf16x3 person=%d/%d, "
              "candidates=%d differing=%d (%.3f %%)" % (B, int(r3["count"].sum()), int(r16["count"].sum()), matched,
                                                        persons, tot, flips, 100.0 * flips / max(tot, 1)))
