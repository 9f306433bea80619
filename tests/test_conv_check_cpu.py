"""CPU: the conv-level checker of tests/plan_check.py (conv_op, check_conv, conv_mutations) on float64 CPU tensors, so
that the checker the GPU sweep relies on (tests/test_conv_edges_gpu.py) is itself checked without a GPU.  A synthetic
device output - the float64 reference of the device's operands, rounded as the device stores it - must pass in every
precision and epilogue form, and every wrong reference that applies must be flagged."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import (_K, _X3_ONLY, check_conv, conv_inputs, conv_mutations, conv_op, conv_operands,  # noqa: E402
                        device_planes, f32_out, reference, value)

OPS = {
    "conv3x3_long_k": conv_op(1, 3, 4, 1024, 64, k=3),
    "conv1x1_s2_odd": conv_op(1, 7, 9, 128, 96, k=1, s=2),
    "residual_norelu": conv_op(1, 5, 6, 64, 64, k=3, relu=False, res=True),
    "res_p1_p2": conv_op(2, 3, 5, 256, 64, res=True, posts=2),
    "pair_s1": conv_op(1, 4, 5, 128, 64, cin2=64, s2=1),
    "pair_s2": conv_op(1, 4, 5, 64, 64, cin2=256, s2=2),
    "up_from_3x2": conv_op(1, 6, 4, 128, 64, up=True),
    "f32_c14": conv_op(1, 5, 7, 128, 14, k=3, relu=False, f32=True),
}


def _stored(r, op, precision):
    """What the device would store for the exact value r: fp32 for fp32 outputs, else the precision's planes of fp32(r)
    (the fp32 epilogue value), read back as their sum."""
    v = r.float()
    return v.double() if f32_out(op) else value(device_planes(v, precision))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16", "fp16"])
@pytest.mark.parametrize("name", list(OPS))
def test_checker_passes_the_device_rounding_and_flags_every_wrong_reference(name, precision):
    op = OPS[name]
    t = conv_inputs(op, 3, device="cpu")
    get, get_lo, rw = conv_operands(op, t, precision)
    r = reference(op, get, rw, None, get_lo=get_lo)[0]
    muts = conv_mutations(op, precision)
    j = check_conv(op, _stored(r, op, precision).float(), t, precision, muts=muts)
    assert not j["bad"], j["bad"]
    assert j["err"] <= 1.0 and j["share"] == 0.0
    assert "drop_last_kb" in muts and ("bias_shift" in muts) == (int(op["cout"]) >= 64)
    assert set(_X3_ONLY) <= set(muts) or precision != "bf16x3"
    assert set(j["tried"]) == set(muts), "wrong references equal to the right one: %s" % sorted(set(muts) - set(j["tried"]))
    missed = sorted(m for m, (flagged, _) in j["tried"].items() if not flagged)
    assert not missed, "accepted on %s (K %d): %s" % (name, _K(op), missed)


def test_the_last_k_block_is_the_last_tap_and_the_second_input():
    """drop_last_kb removes exactly the products of the kernel's last k-block: tap (kh - 1, kw - 1), channels Cin - 64 ..
    Cin - 1 of a single input; the last 64 channels of in2 of a K-concatenated pair."""
    for op, role, cin in ((conv_op(1, 4, 4, 128, 32, k=3, relu=False), "in", 128),
                          (conv_op(1, 4, 4, 64, 32, cin2=128, s2=2, relu=False), "in2", 128)):
        t = conv_inputs(op, 4, device="cpu")
        get, _, rw = conv_operands(op, t, "bf16")
        r = reference(op, get, rw, None)[0]
        rm = reference(op, get, rw, None, mut="drop_last_kb")[0]
        t[role][..., cin - 64:] = 0  # the same channels zeroed in the input instead
        get0, _, _ = conv_operands(op, t, "bf16")
        r0 = reference(op, get0, rw, None)[0]
        assert not torch.equal(rm, r)
        if role == "in2":  # a 1x1 input: its last 64 channels are the whole last k-block
            assert torch.allclose(rm, r0, rtol=0, atol=1e-12)
        else:  # of a 3x3 input only the bottom-right tap goes: the output pixel whose tap (2, 2) is out of bounds keeps r
            assert torch.equal(rm[:, -1, -1], r[:, -1, -1]) and not torch.equal(rm[:, 0, 0], r[:, 0, 0])
