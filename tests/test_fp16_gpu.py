"""GPU: the fp16 precision (SMAPB_PREC_FP16): fp16 operands and activations, fp32 accumulation, stores clamped to +-65504.

  * single convolutions (the CASES of tests/test_conv_gpu.py) against a float64 reference built from the fp16-rounded
    operands the device holds: |y - r| <= 1/2 ulp_fp16(y) + _acc_bound (tests/test_plan_ops_gpu.py), and the same checker
    flags a reference built from bf16-rounded operands;
  * saturation: outputs beyond +-65504 are exactly +-65504, never inf / NaN, and counted; folded weights beyond the range
    are rejected by finalize;
  * every op of the real plan against a float64 reference of its own layer, as tests/test_plan_ops_gpu.py does for bf16x3
    and bf16, and plan switches that must not change a bit;
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
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import smap_torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_conv_gpu import CASES  # noqa: E402
from test_plan_ops_gpu import _acc_bound, _consumers, _K, _nchw, _nhwc, op_class, plan_ops, reference, x3_error  # noqa: E402

pytestmark = pytest.mark.gpu

FP16_MAX = 65504.0
FP16_BOUND = 1e-2  # backbone vs fp32 oracle, max|a - b| / max|ref| per tensor (measured <= 4.99e-3, see above)
SEED = 5


def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def half_ulp16(y):
    """Half an fp16 ulp of fp16 values y (fp64 tensor): the round-to-nearest error of the store that produced them."""
    a = y.abs()
    _, e = torch.frexp(a)  # a = m 2^e, m in [0.5, 1): ulp = 2^(e - 1 - 10), subnormal ulp 2^-24
    e = torch.clamp(e - 11, min=-24)
    return torch.ldexp(torch.full_like(a, 0.5), e)


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    _no_tf32()
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


def _case_tensors(case):
    B, H, W, Cin, Cout, k, stride, relu, use_res = case
    g = torch.Generator(device="cpu").manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    res = torch.randn(B, Ho, Wo, Cout, generator=g).cuda() if use_res else None
    return x, w, b, res


def _conv_reference(case, x, w, b, res, rnd):
    """fp64 (r, pre, q) of one conv_test case with x, w, res rounded by rnd (the device's storage format)."""
    B, H, W, Cin, Cout, k, stride, relu, use_res = case
    d = lambda t: rnd(t).double()  # noqa: E731
    conv = lambda xx, ww: F.conv2d(_nchw(xx), ww, stride=stride, padding=k // 2)  # noqa: E731
    pre = _nhwc(conv(d(x), d(w))) + b.double()
    sq = _nhwc(conv(d(x) ** 2, d(w) ** 2)) + b.double() ** 2
    if use_res:
        pre = pre + d(res)
        sq = sq + d(res) ** 2
    r = F.relu(pre) if relu else pre
    return r, pre, sq.sqrt()


def _conv_op(case):
    return {"kind": "conv", "k": "%dx%d" % (case[5], case[5]), "cin": str(case[3])}


@pytest.mark.parametrize("case", CASES)
def test_conv_fp16_matches_fp64_of_device_operands(eng, case):
    x, w, b, res = _case_tensors(case)
    relu = case[7]
    y = eng.conv_test(x, w, b, res=res, stride=case[6], relu=relu, precision="fp16").double()
    torch.cuda.synchronize()
    assert torch.equal(y, y.half().double()), "outputs are not fp16 values"
    r, pre, q = _conv_reference(case, x, w, b, res, lambda t: t.half())
    bound = half_ulp16(y) + _acc_bound(_conv_op(case), q, r, pre)
    err = ((y - r).abs() / bound).max().item()
    assert err <= 1.0, "error %.3g x the bound" % err
    if relu:  # the ReLU clears exactly
        assert (y[pre < -_acc_bound(_conv_op(case), q, pre)] == 0).all()
    assert eng.saturation_count(reset=True) == 0


def test_checker_flags_a_bf16_operand_reference(eng):
    """On the largest-K case the checker that passes fp16 rejects a reference built from bf16-rounded operands: the bound
    resolves fp16's 4x finer operand rounding."""
    case = max(CASES, key=lambda c: c[3] * c[5] * c[5])
    x, w, b, res = _case_tensors(case)
    y = eng.conv_test(x, w, b, res=res, stride=case[6], relu=case[7], precision="fp16").double()
    r16, pre16, q = _conv_reference(case, x, w, b, res, lambda t: t.half())
    r, pre, _ = _conv_reference(case, x, w, b, res, lambda t: t.bfloat16())
    over16 = (y - r16).abs() > half_ulp16(y) + _acc_bound(_conv_op(case), q, r16, pre16)
    over = (y - r).abs() > half_ulp16(y) + _acc_bound(_conv_op(case), q, r, pre)
    print("\n[fp16 checker] K=%d: fp16-operand reference %.3g, bf16-operand reference %.3g of the elements outside the"
          " bound" % (_K(_conv_op(case)), over16.double().mean().item(), over.double().mean().item()))
    assert not over16.any()
    assert over.double().mean().item() > 0.05


_TILE_CASES = [(8, 32, 52, 256, 256, 3, 1, False), (8, 32, 52, 1024, 256, 1, 1, False), (2, 16, 26, 512, 512, 3, 2, False),
               (4, 64, 104, 128, 512, 1, 1, True), (2, 128, 208, 256, 64, 1, 1, False)]


@pytest.mark.parametrize("case", _TILE_CASES)
def test_fp16_every_tile_width_and_every_run_gives_the_same_bits(eng, monkeypatch, case):
    B, H, W, Cin, Cout, k, stride, use_res = case
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    res = torch.randn(B, Ho, Wo, Cout, generator=g).cuda() if use_res else None
    first, n = None, 0
    for tile in ("128,1", "64,1", "32,1"):
        if Cout % int(tile.split(",")[0]):
            continue
        monkeypatch.setenv("SMAPB_FORCE_TILE", tile)
        for _ in range(2):
            y = eng.conv_test(x, w, b, res=res, stride=stride, relu=True, precision="fp16")
            torch.cuda.synchronize()
            if first is None:
                first = y
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

    sd = smap_torch.make_state_dict(0, "identity")
    unit = "stage1.downsample.layer2.1.conv_bn_relu2"
    sd[unit + ".conv.weight"] = sd[unit + ".conv.weight"].clone()
    sd[unit + ".conv.weight"][3, 1, 0, 0] = 1.0e5
    e = Engine(0, max_batch=1, in_h=64, in_w=96)
    try:
        with pytest.raises(SmapB200Error, match=unit.replace(".", r"\.")):
            e.load_state_dict(sd, "fp16")
        x = smap_torch.make_input(1, 64, 96, seed=1).cuda()
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


class Weights16:
    """Per-unit (W, bias, None) as the device holds them in fp16: folded in float64, rounded to fp32 (fold_unit), weights
    rounded to fp16, biases fp32."""

    mode = "fp16"

    def __init__(self, sd):
        self.sd, self.cache = sd, {}

    def unit(self, name):
        if name not in self.cache:
            g = lambda k: self.sd[name + k].double().cuda()  # noqa: E731
            s = g(".bn.weight") / torch.sqrt(g(".bn.running_var") + smap_torch.BN_EPS)
            W = (g(".conv.weight") * s.view(-1, 1, 1, 1)).float().half().double()
            bias = ((g(".conv.bias") - g(".bn.running_mean")) * s + g(".bn.bias")).float()
            self.cache[name] = (W, bias, None)
        return self.cache[name]

    def bias_sum(self, b1, b2):
        return (b1 + b2).double()


def _dims(op):
    return [int(v) for v in op["out"].split("x")]


def dump16(eng, B, op):
    """Op output on the device: fp16 [N, H, W, C] or fp32 [N, H, W, C] (heads)."""
    N, H, W, C = _dims(op)
    t = torch.empty(N, H, W, C, dtype=torch.float32 if op["kind"] == "conv_f32" else torch.float16, device="cuda")
    nbytes = t.numel() * t.element_size()
    got = eng.lib.smapb_debug_dump(eng._h, B, op["idx"], ctypes.c_void_p(t.data_ptr()), nbytes, 0)
    assert got == nbytes, (op["name"], got, nbytes)
    return t


def _s2d_expected16(img):
    N, _, H, W = img.shape
    v = img.reshape(N, 3, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(N, H // 2, W // 2, 12)
    return F.pad(v, (0, 4, 2, 1)).half()


def check_plan16(H, W, B):
    from smap_b200.engine import Engine

    _no_tf32()
    print("\n[plan ops fp16 %dx%d B=%d]" % (H, W, B))
    sd = smap_torch.make_state_dict(SEED, "random")
    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    worst, failures = {}, []
    try:
        eng.load_state_dict(sd, "fp16")
        eng.forward(smap_torch.make_input(B, H, W, seed=SEED + 1).cuda())
        img = smap_torch.make_input(B, H, W, seed=SEED + 2).cuda()
        eng.forward(img)
        torch.cuda.synchronize()
        _, ops = plan_ops(eng, B)
        wts = Weights16(sd)
        uses = _consumers(ops)
        live = {}
        for op in ops:
            i, cls = op["idx"], op_class(op)
            if op["kind"] != "conv_f32" and op.get("dtype") != "f16":
                failures.append("op %d %s: description lacks dtype=f16" % (i, op["name"]))
            y_raw = dump16(eng, B, op)
            if uses.get(i):
                live[i] = y_raw
            get = lambda role: live[int(op[role])].double()  # noqa: E731
            if op["kind"] == "s2d":
                ok = torch.equal(y_raw, _s2d_expected16(img))
                err, bad = (0.0 if ok else math.inf), ([] if ok else ["s2d not bit-exact"])
            elif op["kind"] == "maxpool":
                ok = torch.equal(y_raw.double(), _nhwc(F.max_pool2d(_nchw(get("a")), 3, 2, 1)))
                err, bad = (0.0 if ok else math.inf), ([] if ok else ["max-pool not bit-exact"])
            else:
                y = y_raw.double()
                r, pre, relu_last = reference(op, get, wts, img)
                q = reference(op, get, wts, img, squares=True)[0].sqrt()
                out_round = (lambda t: t.abs() * 2.0 ** -24) if op["kind"] == "conv_f32" else half_ulp16
                bound = out_round(y[..., :r.shape[-1]]) + _acc_bound(op, q, r, pre)
                _, bad = x3_error(y, r, pre, relu_last, neg=_acc_bound(op, q, pre))
                err = ((y[..., :r.shape[-1]] - r).abs() / bound.clamp(min=1e-30)).max().item()
                if err > 1.0:
                    bad.append("error %.3g x the bound" % err)
                if op["kind"] != "conv_f32" and not torch.isfinite(y).all():
                    bad.append("non-finite activations")
            worst[cls] = max(worst.get(cls, 0.0), err)
            if bad:
                failures.append("op %d %s (%s, bn %s, tw %s): %s" % (i, op["name"], cls, op.get("bn"), op.get("tw"),
                                                                    "; ".join(bad)))
            for j in [int(op[r]) for r in ("in", "in2", "res", "p1", "p2", "up", "a", "b") if r in op and op[r] != "x"]:
                uses[j].remove(i)
                if not uses[j]:
                    live.pop(j, None)
        assert eng.saturation_count() == 0
    finally:
        eng.close()
    torch.cuda.empty_cache()
    for k in sorted(worst):
        print("  %-22s %.3g" % (k, worst[k]))
    return ops, failures


@pytest.mark.parametrize("geom", PLAN_GEOMS, ids=lambda g: "%dx%d_b%d" % g)
def test_plan_ops_fp16(geom):
    ops, failures = check_plan16(*geom)
    assert not failures, "\n".join(failures)
    seen = {op_class(o) for o in ops}
    for need in ("conv1x1", "conv3x3", "residual", "fused_pair_s1", "fused_pair_s2", "up_residual", "res_p1_p2", "head_f32",
                 "tapexp", "stem_tc", "maxpool", "s2d"):
        assert need in seen, "no %s op checked (seen: %s)" % (need, sorted(seen))


def _run_sums16(H, W, B, sd, x):
    from smap_b200.engine import Engine

    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, "fp16")
        outs = [o.cpu() for o in eng.forward(x)]
        torch.cuda.synchronize()
        sums, ops = plan_ops(eng, B)
    finally:
        eng.close()
    return sums, ops, outs


@pytest.mark.parametrize("geom", [(64, 96, 2), (512, 832, 2)], ids=lambda g: "%dx%d_b%d" % g)
def test_fp16_plan_switches_keep_the_bits(geom, monkeypatch):
    from smap_b200 import _lib
    from smap_b200.engine import get_tile_table

    H, W, B = geom
    sd = smap_torch.make_state_dict(SEED, "random")
    x = smap_torch.make_input(B, H, W, seed=SEED + 3).cuda()
    base_sums, base_ops, base_outs = _run_sums16(H, W, B, sd, x)

    def same(tag, sums, ops, outs):
        assert [o["name"] for o in ops] == [o["name"] for o in base_ops], tag
        diff = [o["name"] for o, a, b in zip(ops, sums, base_sums) if a != b]
        assert not diff, "%s: %d ops differ from the default plan, first %s" % (tag, len(diff), diff[:3])
        for a, b in zip(outs, base_outs):
            assert torch.equal(a, b), tag

    for var in ("SMAPB_SERPENTINE", "SMAPB_PDL", "SMAPB_ONE_STREAM"):
        with monkeypatch.context() as m:
            m.setenv(var, "1")
            same(var, *_run_sums16(H, W, B, sd, x))
    lib = _lib.load()
    table = get_tile_table()
    assert any(line.split("\t")[0].endswith(" f16") for line in table.splitlines())  # fp16 rows of their own
    try:
        for bn in (32, 64, 128):
            forced = []
            for line in table.splitlines():
                key, tbn, cg = line.split("\t")
                if int(key.split("/")[1]) % bn == 0:
                    tbn = str(bn)
                forced.append("\t".join((key, tbn, cg)))
            lib.smapb_set_tile_table("\n".join(forced).encode() + b"\n")
            with monkeypatch.context() as m:
                m.setenv("SMAPB_FORCE_TILE", str(bn))
                m.setenv("SMAPB_NO_AUTOTUNE", "1")
                same("SMAPB_FORCE_TILE=%d" % bn, *_run_sums16(H, W, B, sd, x))
    finally:
        lib.smapb_set_tile_table(table.encode())


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
    _no_tf32()
    ref = smap_torch.smap_forward(sd_dev, x)
    torch.backends.cudnn.allow_tf32 = True  # PyTorch's default: the reference's own SMAP.cuda() convolutions
    tf32 = smap_torch.smap_forward(sd_dev, x)
    _no_tf32()
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

    _no_tf32()
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
