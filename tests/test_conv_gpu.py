"""GPU: the wgmma implicit-GEMM convolution against a plain PyTorch fp32 reference of the same op
(TF32 disabled).  Tolerance for the bf16x3 (split-bf16, fp32-faithful) mode: 2e-5 of the output max."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_check import CASES, _TILE_CASES, _case_tensors, no_tf32  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    no_tf32()
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


@pytest.mark.parametrize("case", CASES)
def test_conv_bf16x3_matches_fp32(eng, case):
    B, H, W, Cin, Cout, k, stride, relu, use_res = case
    x, w, b, res = _case_tensors(case)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=stride, padding=k // 2)
    if use_res:
        ref = ref + res.permute(0, 3, 1, 2)
    if relu:
        ref = F.relu(ref)
    y = eng.conv_test(x, w, b, res=res, stride=stride, relu=relu)
    torch.cuda.synchronize()
    ref = ref.permute(0, 2, 3, 1)
    err = (y - ref).abs().max().item() / ref.abs().max().item()
    assert err < 2e-5, "relative error %g" % err


def test_conv_bf16_fast_mode_is_coarser_but_sane(eng):
    g = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn(1, 16, 24, 128, generator=g).cuda()
    w = (torch.randn(128, 128, 3, 3, generator=g) / (128 * 9) ** 0.5).cuda()
    b = torch.zeros(128).cuda()
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, padding=1).permute(0, 2, 3, 1)
    y = eng.conv_test(x, w, b, relu=False, precision="bf16")
    err = (y - ref).abs().max().item() / ref.abs().max().item()
    assert err < 2e-2


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 128, 208, 64, 256), (8, 64, 104, 128, 512), (1, 16, 26, 512, 2048)])
def test_conv_residual_and_post_adds_deterministic(eng, B, H, W, Cin, Cout):
    """Last bottleneck of a layer in stages 1-2: relu(conv3 + x) + skip1 + skip2 (model/smap.py:74-75,143)."""
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    res, p1, p2 = (torch.randn(B, H, W, Cout, generator=g).cuda() for _ in range(3))
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2), w, b).permute(0, 2, 3, 1) + res) + p1 + p2
    ys = [eng.conv_test(x, w, b, res=res, relu=True, post1=p1, post2=p2) for _ in range(4)]
    torch.cuda.synchronize()
    for y in ys:
        assert torch.equal(y, ys[0]), "non-deterministic output"
        assert (y - ref).abs().max().item() / ref.abs().max().item() < 2e-5


_TILES = ("128", "64", "32")


@pytest.mark.parametrize("case", _TILE_CASES)
def test_every_tile_shape_gives_the_same_bits(eng, monkeypatch, case):
    """The tile table / autotuner may pick any of these BLOCK_N shapes: each must be correct AND all must
    produce the same bits (every output element accumulates its K products in the same order whatever the tile), so that
    results do not depend on which shape a handle, a process or a rank happens to use."""
    B, H, W, Cin, Cout, k, stride, use_res = case
    x, w, b, res = _case_tensors(case, seed=11)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    ref = F.relu(ref + res if use_res else ref)
    first, n = None, 0
    for tile in _TILES:
        bn = int(tile)
        if Cout % bn:
            continue
        monkeypatch.setenv("SMAPB_FORCE_TILE", tile)
        y = eng.conv_test(x, w, b, res=res, stride=stride, relu=True)
        torch.cuda.synchronize()
        err = (y - ref).abs().max().item() / ref.abs().max().item()
        assert err < 2e-5, "tile %s: relative error %g" % (tile, err)
        if first is None:
            first = y
        assert torch.equal(y, first), "tile %s differs from tile %s in %d elements" % (tile, _TILES[0], (y != first).sum().item())
        n += 1
    assert n >= 2
