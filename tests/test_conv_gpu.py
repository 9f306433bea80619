"""GPU: the wgmma implicit-GEMM convolution against a plain PyTorch fp32 reference of the same op
(TF32 disabled).  Tolerance for the bf16x3 (split-bf16, fp32-faithful) mode: 2e-5 of the output max."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    e = Engine(0, max_batch=2, in_h=64, in_w=96)
    yield e
    e.close()


CASES = [
    # B, H, W, Cin, Cout, k, stride, relu, res
    (1, 16, 24, 64, 64, 1, 1, True, False),      # flat 1x1, single k-block
    (2, 16, 26, 256, 64, 1, 1, True, False),     # flat 1x1, ragged M (832 rows)
    (1, 16, 24, 64, 256, 1, 1, False, True),     # residual epilogue, N=256
    (2, 32, 52, 128, 128, 3, 1, True, False),    # 3x3 s1, patch tiles, padding via TMA OOB
    (1, 16, 26, 512, 512, 3, 1, True, False),    # 3x3 s1 on the 16x26 level (non power-of-two width)
    (2, 32, 52, 128, 128, 3, 2, True, False),    # 3x3 stride 2 (TMA elementStrides)
    (1, 64, 104, 256, 512, 1, 2, False, False),  # 1x1 stride 2 (downsample branch)
    (1, 32, 52, 256, 43, 3, 1, False, False),    # thin head, Cout padded to 64
    (1, 32, 52, 256, 14, 3, 1, False, False),    # thin head, Cout padded to 32
    (1, 16, 24, 256, 1, 3, 1, False, False),     # root-depth head
    (2, 16, 26, 2048, 512, 1, 1, True, False),   # long K (32 k-blocks): ring wrap-around
    # persistent regime: many tiles per CTA (accumulator / residual / staging rings wrap many times)
    (8, 128, 208, 64, 256, 1, 1, True, True),    # layer1 conv3 + residual, 3328 tiles
    (8, 128, 208, 256, 64, 1, 1, True, False),   # N=64 tiles, 2 chunks
    (4, 128, 208, 64, 64, 3, 1, True, False),    # 3x3 patch tiles, 832 tiles
    (8, 64, 104, 128, 512, 1, 1, False, True),   # layer2 conv3 + residual
    (8, 128, 208, 256, 14, 3, 1, False, False),  # N=32 single-chunk tiles (one epilogue group idle)
]


@pytest.mark.parametrize("case", CASES)
def test_conv_bf16x3_matches_fp32(eng, case):
    B, H, W, Cin, Cout, k, stride, relu, use_res = case
    g = torch.Generator(device="cpu").manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    pad = k // 2
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=stride, padding=pad)
    res = None
    if use_res:
        res = torch.randn(B, ref.shape[2], ref.shape[3], Cout, generator=g).cuda()
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


_TILE_CASES = [(8, 32, 52, 256, 256, 3, 1, False), (8, 32, 52, 1024, 256, 1, 1, False), (2, 16, 26, 512, 512, 3, 2, False),
               (4, 64, 104, 128, 512, 1, 1, True), (2, 128, 208, 256, 64, 1, 1, False)]
_TILES = ("128,1", "64,1", "32,1")


@pytest.mark.parametrize("case", _TILE_CASES)
def test_every_tile_shape_gives_the_same_bits(eng, monkeypatch, case):
    """The tile table / autotuner may pick any of these BLOCK_N shapes: each must be correct AND all must
    produce the same bits (every output element accumulates its K products in the same order whatever the tile), so that
    results do not depend on which shape a handle, a process or a rank happens to use."""
    B, H, W, Cin, Cout, k, stride, use_res = case
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda()
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
    res = torch.randn(ref.shape, generator=g).cuda() if use_res else None
    ref = F.relu(ref + res if use_res else ref)
    first, n = None, 0
    for tile in _TILES:
        bn = int(tile.split(",")[0])
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
