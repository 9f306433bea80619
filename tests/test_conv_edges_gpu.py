"""GPU: every instance of the tensor-core convolution, conv_tc_kernel<BLOCK_N in {128, 64, 32}, NTERMS, RING in {0, 1, 2},
E> in bf16x3, bf16 and fp16 (27 instances), driven through smapb_conv_test at the edges where tiled kernels break, each
output element held to the per-element float64 bound the plan's ops meet (judge() in tests/plan_check.py).

The cases are chosen from the kernel and its set-up, not from the network:
  * flat 1x1 convs (one row of 128-pixel tiles) with N*Ho*Wo of 1, 127, 128, 129, one short of and one past a wave of
    132 tiles, and one past two waves: a lone partial tile, one tile per CTA with the second consumer warpgroup idle, a
    ragged last wave and unequal tile counts between the two consumer warpgroups;
  * patch tiles of every width tw in {1, ..., 128} that patch_width picks, with Ho and Wo not multiples of the patch,
    stride 2 on odd inputs, and 3x3 on 1x1, 1xN and Nx1 images (every tap but the centre is out-of-bounds fill);
  * K from one k-block (the operand ring never fills) to 288 (Cin 2048, 3x3), M kept small where K is large;
  * Cout in {1, 14, 32, 43, 64, 96, 160, 256}: 96 and 160 are odd numbers of 32-channel chunks and force BLOCK_N 32,
    with RING 0 and 1;
  * every epilogue form: residual without ReLU, residual + two skips, the K-concatenated pair with stride2 1 and 2, the
    bilinear up-residual from 1x1, 1xN, 2x2, 13x7, 40x1, 33x3 and 3x33 maps (the last row and column take the clamped i1),
    and fp32 outputs (the heads' store) for Cout 1, 14, 43 and 126.
Every case runs in all three precisions at every tile width that divides Cout_pad (SMAPB_FORCE_TILE), and twice: all
widths and both runs give the same bits, and in fp16 the saturation count stays 0 (the inputs are in range).
`-s` prints the worst |y - r| / bound per instance, and for every wrong reference of conv_mutations the share of
elements outside the bound on the largest-K case of each epilogue form."""
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import (_K, _dims, check_conv, conv_inputs, conv_mutations, conv_op, f32_out, no_tf32, op_class,  # noqa: E402
                        run_conv)

pytestmark = pytest.mark.gpu

PRECISIONS = ("bf16x3", "bf16", "fp16")
WIDTHS = (128, 64, 32)
WAVE = 132 * 128  # output pixels of one wave of 128-pixel tiles on the H100's 132 SMs
TWS = (1, 2, 4, 8, 16, 32, 64, 128)

CASES = {
    # flat 1x1 (is_flat): N*Ho*Wo around one tile and one or two waves
    "flat_m1": conv_op(1, 1, 1, 64, 64),
    "flat_m127": conv_op(1, 1, 127, 64, 32),
    "flat_m128": conv_op(2, 8, 8, 64, 128),
    "flat_m129": conv_op(1, 3, 43, 64, 256),
    "flat_wave_minus_1": conv_op(5, 31, 109, 64, 32),  # WAVE - 1
    "flat_wave_plus_1": conv_op(1, 61, 277, 64, 128),  # WAVE + 1
    "flat_2waves_plus_1": conv_op(1, 47, 719, 64, 64),  # 2 WAVE + 1
    # patch tiles: one geometry per tw patch_width picks, partial patches, stride 2 on odd inputs, 1-pixel sides
    "tw1_130x1": conv_op(1, 130, 1, 64, 64, k=3),
    "tw2_67x2": conv_op(1, 67, 2, 64, 32, k=3),
    "tw4_67x3": conv_op(1, 67, 3, 128, 64, k=3),
    "tw8_s2_17x9": conv_op(2, 17, 9, 64, 64, k=3, s=2),
    "tw16_7x1": conv_op(1, 7, 1, 64, 32, k=3),
    "tw16_s2_13x27_c96": conv_op(1, 13, 27, 64, 96, k=3, s=2),
    "tw32_9x17": conv_op(1, 9, 17, 64, 64, k=3),
    "tw32_s2_25x51": conv_op(1, 25, 51, 128, 32, k=3, s=2),
    "tw64_5x33_c160": conv_op(1, 5, 33, 64, 160, k=3),
    "tw64_s2_3x257": conv_op(1, 3, 257, 64, 64, k=3, s=2),
    "tw128_1x1": conv_op(2, 1, 1, 64, 64, k=3),
    "tw128_1x7_c43": conv_op(1, 1, 7, 64, 43, k=3),
    "tw128_1x200_c14": conv_op(1, 1, 200, 64, 14, k=3),
    "ds_1x1_s2_11x21": conv_op(1, 11, 21, 128, 256, k=1, s=2),
    # K
    "k1_s2_c1": conv_op(1, 5, 9, 64, 1, k=1, s=2, relu=False),
    "k16_flat": conv_op(1, 4, 33, 1024, 256),
    "k288_3x3": conv_op(1, 3, 5, 2048, 64, k=3),
    # epilogue forms (RING 1: residual and skips; odd chunk counts force BLOCK_N 32)
    "res_norelu_c96": conv_op(1, 9, 17, 64, 96, k=3, relu=False, res=True),
    "res_norelu_flat": conv_op(1, 8, 129, 64, 64, relu=False, res=True),
    "res_p1_p2_c160": conv_op(1, 6, 11, 128, 160, res=True, posts=2),
    "res_p1_p2_3x3": conv_op(2, 7, 9, 256, 128, k=3, res=True, posts=2),
    "res_p1_p2_k144": conv_op(1, 2, 3, 1024, 64, k=3, res=True, posts=2),
    "pair_s1": conv_op(1, 6, 7, 128, 256, cin2=64, s2=1),
    "pair_s2": conv_op(2, 5, 9, 64, 128, cin2=256, s2=2),
    "pair_s2_k24": conv_op(1, 3, 4, 512, 64, cin2=1024, s2=2),
    # RING 2: the up-residual, low-resolution maps 1x1, 1x5, 2x2, 13x7, 40x1 and 33x3
    "up_from_1x1": conv_op(1, 2, 2, 64, 64, up=True),
    "up_from_1x5": conv_op(1, 2, 10, 64, 32, up=True),
    "up_from_2x2": conv_op(1, 4, 4, 128, 64, up=True, relu=False),
    "up_from_13x7": conv_op(2, 26, 14, 64, 128, up=True),
    "up_from_40x1": conv_op(1, 80, 2, 64, 32, up=True),
    "up_from_33x3_3x3": conv_op(1, 66, 6, 64, 64, k=3, up=True),
    "up_from_3x33_k72": conv_op(1, 6, 66, 512, 64, k=3, up=True),
    # fp32 outputs, as the heads store them
    "f32_c1": conv_op(1, 16, 24, 256, 1, k=3, relu=False, f32=True),
    "f32_c14": conv_op(1, 9, 13, 128, 14, k=3, relu=False, f32=True),
    "f32_c43": conv_op(1, 7, 9, 64, 43, k=3, relu=False, f32=True),
    "f32_c126_flat": conv_op(1, 5, 7, 256, 126, relu=False, f32=True),
}


def _seed(name):
    return sum(ord(c) * (i + 1) for i, c in enumerate(name)) % (2 ** 31)


def _form(op):
    return "f32" if f32_out(op) else op_class(op)


def _widths(op):
    cout_pad = (int(op["cout"]) + 31) // 32 * 32
    return [bn for bn in WIDTHS if cout_pad % bn == 0]


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    no_tf32()
    e = Engine(0, max_batch=1, in_h=64, in_w=96)
    yield e
    e.close()


_RUNS = {}


def _largest_k_per_form():
    best = {}
    for name, op in CASES.items():
        f = _form(op)
        if f not in best or _K(op) > _K(CASES[best[f]]):
            best[f] = name
    return best


def _run(eng, name, precision):
    """Run case `name` in `precision` at every legal width, twice each, and check the first output (once per session per
    case and precision; on the largest-K case of its epilogue form with the wrong references of conv_mutations too).
    -> dict err (|y - r| / bound), launches (the reported launch of every run), bad (failures), muts and tried (judge's),
    seconds."""
    key = (name, precision)
    if key in _RUNS:
        return _RUNS[key]
    op = CASES[name]
    muts = conv_mutations(op, precision) if name in _largest_k_per_form().values() else []
    t0 = time.time()
    t = conv_inputs(op, _seed(name))
    first, launches, err, bad, tried = None, [], None, [], {}
    mp = pytest.MonkeyPatch()
    try:
        for bn in _widths(op):
            mp.setenv("SMAPB_FORCE_TILE", str(bn))
            for rep in range(2):
                launch = {}
                y = run_conv(eng, op, t, precision, launch)
                torch.cuda.synchronize()
                launches.append(launch)
                if launch["block_n"] != bn:
                    bad.append("SMAPB_FORCE_TILE=%d ran block_n %d" % (bn, launch["block_n"]))
                if precision == "fp16":
                    n = eng.saturation_count(reset=True)
                    if n:
                        bad.append("width %d run %d: saturation count %d" % (bn, rep, n))
                    if not f32_out(op) and not torch.equal(y, y.half().float()):
                        bad.append("width %d: outputs are not fp16 values" % bn)
                if first is None:
                    first = y
                    j = check_conv(op, y, t, precision, muts=muts)
                    bad += j["bad"]
                    err, tried = j["err"], j["tried"]
                elif not torch.equal(y, first):
                    bad.append("width %d run %d: %d elements differ from width %d run 0"
                               % (bn, rep, int((y != first).sum().item()), _widths(op)[0]))
    finally:
        mp.undo()
    _RUNS[key] = {"op": op, "err": err, "launches": launches, "bad": bad, "muts": muts, "tried": tried,
                  "s": time.time() - t0}
    return _RUNS[key]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(CASES))
def test_conv_edge_case(eng, name, precision):
    """Within the bound at one width, the same bits at every width and on a second run."""
    r = _run(eng, name, precision)
    l0 = r["launches"][0]
    print("\n[conv %s %s] K %d tw %d %s ring %d: |y - r| / bound %.3g, widths %s, %.2f s"
          % (name, precision, _K(r["op"]), l0["tw"], "flat" if l0["flat"] else "patch", l0["ring"],
             r["err"], [la["block_n"] for la in r["launches"][::2]], r["s"]))
    assert not r["bad"], "\n".join(r["bad"])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_checker_flags_wrong_references(eng, precision):
    """On the largest-K case of each epilogue form, every wrong reference of conv_mutations that differs from the right
    one puts elements outside the bound (or breaks the exact zeros of the ReLU), while the right one passes."""
    missed, never = [], []
    print("\n[wrong references %s] share of the elements outside the bound" % precision)
    for form, name in sorted(_largest_k_per_form().items()):
        op = CASES[name]
        r = _run(eng, name, precision)
        assert not r["bad"], "\n".join(r["bad"])
        for m in r["muts"]:
            if m not in r["tried"]:
                never.append("%s on %s" % (m, name))
                continue
            flagged, share = r["tried"][m]
            print("  %-14s %-18s K %-6d %-12s %.3g" % (form, name, _K(op), m, share))
            if not flagged:
                missed.append("%s on %s" % (m, name))
    assert not never, "wrong references equal to the right one: %s" % never
    assert not missed, "wrong references the checker accepted: %s" % missed


def test_every_instance_width_and_epilogue_ran(eng):
    """What the launches reported: all 27 (BLOCK_N, precision, RING) instances, every patch width tw in both the flat and
    the patch mode where the kernel has it, and the fp32 output path.  Prints the worst |y - r| / bound per instance."""
    worst, tws, flat_tws, f32 = {}, set(), set(), set()
    for name, op in CASES.items():
        for precision in PRECISIONS:
            r = _run(eng, name, precision)
            for la in r["launches"]:
                inst = (la["block_n"], precision, la["ring"])
                worst[inst] = max(worst.get(inst, 0.0), r["err"])  # every width gave the checked bits
                (flat_tws if la["flat"] else tws).add(la["tw"])
                if f32_out(op):
                    f32.add((la["block_n"], precision))
    print("\n[conv instances] worst |y - r| / bound over the cases each ran")
    for inst in sorted(worst):
        print("  block_n %3d %-6s ring %d  %.3g" % (inst + (worst[inst],)))
    print("  tw patch %s, flat %s; fp32 output at %s" % (sorted(tws), sorted(flat_tws), sorted(f32)))
    want = {(bn, p, ring) for bn in WIDTHS for p in PRECISIONS for ring in (0, 1, 2)}
    assert set(worst) == want, "instances never run: %s" % sorted(want - set(worst))
    assert tws == set(TWS), tws
    assert flat_tws == {128}, flat_tws
    flat_m = {_dims(op)[0] * _dims(op)[1] * _dims(op)[2] for name, op in CASES.items() if name.startswith("flat_")}
    assert flat_m == {1, 127, 128, 129, WAVE - 1, WAVE + 1, 2 * WAVE + 1}, sorted(flat_m)
    assert {p for _, p in f32} == set(PRECISIONS) and {bn for bn, _ in f32} == {32, 64, 128}, sorted(f32)
