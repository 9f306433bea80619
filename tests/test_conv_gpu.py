"""GPU: the wgmma implicit-GEMM convolution at the network's layer shapes, persistent regime included, against the float64
reference of the operands the device holds, element by element: check_conv in tests/plan_check.py, the bound the plan's
ops meet (2^-17 |r| in bf16x3, one bf16 ulp in bf16, plus the accumulation bound; exact zeros where the ReLU clears).
The edges of the tiling, every kernel instance and every epilogue form are swept in tests/test_conv_edges_gpu.py."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import CASES, _TILE_CASES, check_conv, conv_inputs, conv_op, legacy_op, no_tf32, run_conv  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    no_tf32()
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


def _assert_checked(op, y, t, precision):
    j = check_conv(op, y, t, precision)
    assert not j["bad"], "\n".join(j["bad"])
    return j["err"]


@pytest.mark.parametrize("case", CASES)
def test_conv_bf16x3_matches_fp32(eng, case):
    op = legacy_op(case)
    t = conv_inputs(op, hash(case) % (2 ** 31))
    y = run_conv(eng, op, t, "bf16x3")
    torch.cuda.synchronize()
    _assert_checked(op, y, t, "bf16x3")


def test_conv_bf16_fast_mode_is_coarser_but_sane(eng):
    op = conv_op(1, 16, 24, 128, 128, k=3, relu=False)
    t = conv_inputs(op, 0)
    t["b"].zero_()
    y = run_conv(eng, op, t, "bf16")
    torch.cuda.synchronize()
    _assert_checked(op, y, t, "bf16")
    assert not torch.equal(y, run_conv(eng, op, t, "bf16x3")), "bf16 gave the bits of bf16x3"


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 128, 208, 64, 256), (8, 64, 104, 128, 512), (1, 16, 26, 512, 2048)])
def test_conv_residual_and_post_adds_deterministic(eng, B, H, W, Cin, Cout):
    """Last bottleneck of a layer in stages 1-2: relu(conv3 + x) + skip1 + skip2 (model/smap.py:74-75,143)."""
    op = conv_op(B, H, W, Cin, Cout, res=True, posts=2)
    t = conv_inputs(op, 7)
    ys = [run_conv(eng, op, t, "bf16x3") for _ in range(4)]
    torch.cuda.synchronize()
    for y in ys:
        assert torch.equal(y, ys[0]), "non-deterministic output"
    _assert_checked(op, ys[0], t, "bf16x3")


_TILES = ("128", "64", "32")


@pytest.mark.parametrize("case", _TILE_CASES)
def test_every_tile_shape_gives_the_same_bits(eng, monkeypatch, case):
    """The tile table / autotuner may pick any of these BLOCK_N shapes: each must be correct AND all must
    produce the same bits (every output element accumulates its K products in the same order whatever the tile), so that
    results do not depend on which shape a handle, a process or a rank happens to use."""
    op = legacy_op(case)
    t = conv_inputs(op, 11)
    first, n = None, 0
    for tile in _TILES:
        if int(op["cout"]) % int(tile):
            continue
        monkeypatch.setenv("SMAPB_FORCE_TILE", tile)
        launch = {}
        y = run_conv(eng, op, t, "bf16x3", launch)
        torch.cuda.synchronize()
        assert launch["block_n"] == int(tile), launch
        if first is None:
            first = y
            _assert_checked(op, y, t, "bf16x3")
        assert torch.equal(y, first), "tile %s differs from tile %s in %d elements" % (tile, _TILES[0], (y != first).sum().item())
        n += 1
    assert n >= 2
