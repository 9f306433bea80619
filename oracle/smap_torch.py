"""ORACLE - TEST INFRASTRUCTURE ONLY.

Plain-PyTorch fp32 restatement of the reference backbone forward
(model/smap.py:403-419, inference branch) driven directly by the reference's
state-dict schema (SURVEY.md section 8(a), 1876 keys).  It is written as a
functional graph walker, not as a module tree, so it shares no structure with
model/smap.py; parity with the real reference module is pinned by
tests/golden/make_golden.py (which imports /root/reference/model/smap.py in the
build container, runs it on seeded inputs and commits the outputs) and
tests/test_oracle_golden.py.

Also restates the reference's random initialisation (model/smap.py:111-117 +
PyTorch defaults for every other conv) with an explicit generator so that
"random-init SMAP weights" means the same tensors on every box.
"""
import torch
import torch.nn.functional as F

from .schema_ref import (BN_EPS, LAYERS, PLANES, UP_IN, make_input, make_state_dict,  # noqa: F401
                         unit_specs)


# ----------------------------------------------------------------------------
# forward
# ----------------------------------------------------------------------------
def _unit(sd, name, x, stride=1, pad=0, relu=True):
    """conv_bn_relu (model/smap.py:13-45): conv(bias) -> BN(eval) -> optional ReLU."""
    y = F.conv2d(x, sd[name + ".conv.weight"], sd[name + ".conv.bias"], stride=stride, padding=pad)
    y = F.batch_norm(y, sd[name + ".bn.running_mean"], sd[name + ".bn.running_var"],
                     sd[name + ".bn.weight"], sd[name + ".bn.bias"], False, 0.0, BN_EPS)
    return F.relu(y) if relu else y


def _bottleneck(sd, p, x, stride, has_ds):
    """model/smap.py:66-77"""
    out = _unit(sd, p + "conv_bn_relu1", x)
    out = _unit(sd, p + "conv_bn_relu2", out, stride=stride, pad=1)
    out = _unit(sd, p + "conv_bn_relu3", out, relu=False)
    if has_ds:
        x = _unit(sd, p + "downsample", x, stride=stride, relu=False)
    return F.relu(out + x)


def _up(t, size):
    return F.interpolate(t, size=size, mode="bilinear", align_corners=True)


@torch.no_grad()
def smap_forward(sd, imgs, stage_num=3, return_all=False):
    """Inference branch of SMAP.forward (model/smap.py:403-419).

    sd: state dict in the reference schema (tensors on imgs.device, fp32).
    Returns (heatmap_2d [B,43,H/4,W/4], det_d [B,14,..], root_d [B,1,..]).
    """
    B, _, H, W = imgs.shape
    out_shape = (H // 4, W // 4)
    oh, ow = out_shape
    up_sizes = [(oh // 8, ow // 8), (oh // 4, ow // 4), (oh // 2, ow // 2), (oh, ow)]
    x = _unit(sd, "top.conv", imgs, stride=2, pad=3)  # model/smap.py:89
    x = F.max_pool2d(x, 3, 2, 1)  # model/smap.py:90
    skip1 = skip2 = None
    heads = None
    for s in range(stage_num):
        pre = "stage%d." % s
        gen_skip = s != stage_num - 1
        feats = []
        t = x
        for li, nblk in enumerate(LAYERS):  # model/smap.py:140-154
            for b in range(nblk):
                p = "%sdownsample.layer%d.%d." % (pre, li + 1, b)
                t = _bottleneck(sd, p, t, (1 if li == 0 else 2) if b == 0 else 1, b == 0)
            if s > 0:
                t = t + skip1[li] + skip2[li]
            feats.append(t)
        xs = feats[::-1]  # x4, x3, x2, x1
        up_x = None
        res, res_d, res_rd, sk1, sk2 = [], [], [], [], []
        cross = None
        for ind in range(4):  # model/smap.py:210-241
            p = "%supsample.up%d." % (pre, ind + 1)
            out = _unit(sd, p + "u_skip", xs[ind], relu=False)
            if ind > 0:
                u = _up(up_x, up_sizes[ind])
                out = out + _unit(sd, p + "up_conv", u, relu=False)
            out = F.relu(out)
            res.append(_up(_unit(sd, p + "res_conv2", _unit(sd, p + "res_conv1", out), pad=1, relu=False), out_shape))
            res_d.append(_up(_unit(sd, p + "res_d_conv2", _unit(sd, p + "res_d_conv1", out), pad=1, relu=False), out_shape))
            res_rd.append(_up(_unit(sd, p + "res_rd_conv2", _unit(sd, p + "res_rd_conv1", out), pad=1, relu=False), out_shape))
            if gen_skip:
                sk1.append(_unit(sd, p + "skip1", xs[ind]))
                sk2.append(_unit(sd, p + "skip2", out))
                if ind == 3:
                    cross = _unit(sd, p + "cross_conv", out)
            up_x = out
        skip1, skip2 = sk1[::-1], sk2[::-1]  # model/smap.py:281-282 (finest first)
        x = cross
        heads = (res, res_d, res_rd)
    res, res_d, res_rd = heads
    outputs_2d = res[3] + res[2] + res[1]  # model/smap.py:418
    if return_all:
        return outputs_2d, res_d[3], res_rd[3], heads
    return outputs_2d, res_d[3], res_rd[3]


def flip_merge(o2d, o2d_flip):
    """Flip-TTA merge, exps/stage3_root2/test.py:55-70 (SURVEY.md row A7).
    o2d_flip = model(flip(imgs)) BEFORE un-flipping; o2d is modified in place."""
    flip_order = [0, 1, 2, 9, 10, 11, 12, 13, 14, 3, 4, 5, 6, 7, 8]  # data_settings.py:22
    flip_channel = [0, 1, 2, 3, 10, 11, 12, 13, 14, 15, 4, 5, 6, 7, 8, 9,
                    22, 23, 24, 25, 26, 27, 16, 17, 18, 19, 20, 21]  # data_settings.py:33-34
    f = torch.flip(o2d_flip, dims=[-1])
    pair = flip_order + [15 + c for c in flip_channel]
    for i in range(len(pair)):
        if i >= 15 and (i - 15) % 2 == 0:
            o2d[:, i] += f[:, pair[i]] * -1
        else:
            o2d[:, i] += f[:, pair[i]]
    o2d[:, 15:] *= 0.5
    return o2d


def rescale_reference_cuda(hm):
    """exps/stage3_root2/test.py:111-112 as the reference actually executes it: `hmsIn` is a CUDA tensor and ATen's
    CUDA true-divide by a Python scalar multiplies by the fp32 reciprocal (tools/diag_assoc.py);
    a CPU tensor would get an IEEE division.  In place on hm [B,43,h,w]; works on CPU and CUDA tensors alike."""
    r255 = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(255.0, dtype=torch.float32)
    r127 = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(127.0, dtype=torch.float32)
    hm[:, :15] *= r255.to(hm.device)
    hm[:, 15:] *= r127.to(hm.device)
    return hm
