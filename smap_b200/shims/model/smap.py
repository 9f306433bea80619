"""Drop-in replacement for the reference `model.smap` module (model/smap.py): same class name, constructor,
state-dict schema (1876 keys) and inference `forward` contract, backed by libsmap_b200.so.

    from model.smap import SMAP
    model = SMAP(cfg, run_efficient=False); model.to('cuda'); model.load_state_dict(sd); model.eval()
    outputs_2d, outputs_3d, outputs_rd = model(imgs)        # model/smap.py:417-419

Only the inference branch exists (valids/labels must be None): training is out of scope.  Parameters live in
ordinary nn.Conv2d / nn.BatchNorm2d holders so that `.to()`, `.state_dict()`, `.load_state_dict()` behave as in the
reference; they are created in the reference's construction order so that `torch.manual_seed(s); SMAP(cfg)` yields
the same random initialisation (model/smap.py:111-117 re-initialises encoder convs with kaiming_normal_).  The
forward never touches them directly: weights are folded/repacked by the engine (re-synced when they change).
"""
import torch
import torch.nn as nn

from smap_b200.engine import Engine

_LAYERS = (3, 4, 6, 3)
_UP_IN = (2048, 1024, 512, 256)


class _Unit(nn.Module):
    """Parameter holder with the key layout of the reference's conv_bn_relu: .conv.{weight,bias}, .bn.*"""

    def __init__(self, cin, cout, k, stride, pad):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=pad)
        self.bn = nn.BatchNorm2d(cout)


class _Holder(nn.Module):
    pass


def _bottleneck(in_planes, planes, stride, with_ds):
    blk = _Holder()
    ds = _Unit(in_planes, planes * 4, 1, stride, 0) if with_ds else None  # created first (model/smap.py:124-129)
    blk.conv_bn_relu1 = _Unit(in_planes, planes, 1, 1, 0)
    blk.conv_bn_relu2 = _Unit(planes, planes, 3, stride, 1)
    blk.conv_bn_relu3 = _Unit(planes, planes * 4, 1, 1, 0)
    if ds is not None:
        blk.downsample = ds
    return blk


def _encoder():
    enc = _Holder()
    in_planes = 64
    for li, (planes, n) in enumerate(zip((64, 128, 256, 512), _LAYERS)):
        stride = 1 if li == 0 else 2
        blocks = [_bottleneck(in_planes, planes, stride, True)]
        in_planes = planes * 4
        blocks += [_bottleneck(in_planes, planes, 1, False) for _ in range(1, n)]
        setattr(enc, "layer%d" % (li + 1), nn.Sequential(*blocks))
    for m in enc.modules():  # model/smap.py:111-117
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        elif isinstance(m, nn.BatchNorm2d):
            nn.init.constant_(m.weight, 1)
            nn.init.constant_(m.bias, 0)
    return enc


def _up_unit(ind, in_planes, chl, out_chl, gen_skip, gen_cross):
    u = _Holder()
    u.u_skip = _Unit(in_planes, chl, 1, 1, 0)
    if ind > 0:
        u.up_conv = _Unit(chl, chl, 1, 1, 0)
    if gen_skip:
        u.skip1 = _Unit(in_planes, in_planes, 1, 1, 0)
        u.skip2 = _Unit(chl, in_planes, 1, 1, 0)
    if ind == 3 and gen_cross:
        u.cross_conv = _Unit(chl, 64, 1, 1, 0)
    u.res_conv1 = _Unit(chl, chl, 1, 1, 0)
    u.res_conv2 = _Unit(chl, out_chl[0], 3, 1, 1)
    u.res_d_conv1 = _Unit(chl, chl, 1, 1, 0)
    u.res_d_conv2 = _Unit(chl, out_chl[1], 3, 1, 1)
    u.res_rd_conv1 = _Unit(chl, chl, 1, 1, 0)
    u.res_rd_conv2 = _Unit(chl, 1, 3, 1, 1)
    return u


class SMAP(nn.Module):
    def __init__(self, cfg, run_efficient=False, **kwargs):
        super().__init__()
        self.stage_num = cfg.MODEL.STAGE_NUM
        self.kpt_paf_num = cfg.DATASET.KEYPOINT.NUM + cfg.DATASET.PAF.NUM * 2
        self.keypoint_num = cfg.DATASET.KEYPOINT.NUM
        self.paf_num = cfg.DATASET.PAF.NUM
        self.output_shape = cfg.OUTPUT_SHAPE
        self.upsample_chl_num = cfg.MODEL.UPSAMPLE_CHANNEL_NUM
        if self.stage_num != 3 or self.upsample_chl_num != 256 or self.kpt_paf_num != 43 or self.paf_num != 14:
            raise NotImplementedError("smap_b200 implements the stage3_root2 configuration (3 stages, 256 channels, 15+14)")
        self.top = _Holder()
        self.top.conv = _Unit(3, 64, 7, 2, 3)
        for i in range(self.stage_num):
            gen = i != self.stage_num - 1
            st = _Holder()
            st.downsample = _encoder()
            up = _Holder()
            for ind in range(4):
                setattr(up, "up%d" % (ind + 1), _up_unit(ind, _UP_IN[ind], 256, [self.kpt_paf_num, self.paf_num], gen, gen))
            st.upsample = up
            setattr(self, "stage%d" % i, st)
        self.precision = kwargs.get("precision", "bf16x3")
        self._engines = {}
        self._synced = {}

    def _weights_version(self):
        return tuple(p._version for p in self.parameters()) + tuple(b._version for b in self.buffers())

    def forward(self, imgs, valids=None, labels=None, rdepth=None):
        if valids is not None or labels is not None or self.training:
            raise NotImplementedError("smap_b200.SMAP implements the inference branch only (call .eval(); no labels)")
        if not imgs.is_cuda:
            raise RuntimeError("smap_b200.SMAP runs on an H100 only: move the model and the input to 'cuda'")
        B, _, H, W = imgs.shape
        key = (imgs.device.index, H, W)
        eng = self._engines.get(key)
        if eng is None or eng.max_batch < B:
            eng = Engine(imgs.device.index, max_batch=max(B, 8), in_h=H, in_w=W)
            self._engines[key] = eng
            self._synced.pop(key, None)
        ver = self._weights_version()
        if self._synced.get(key) != ver:
            eng.load_state_dict(self.state_dict(), precision=self.precision)
            self._synced[key] = ver
        with torch.cuda.device(imgs.device):
            return eng.forward(imgs.float())
