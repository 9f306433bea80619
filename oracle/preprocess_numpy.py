"""ORACLE - TEST INFRASTRUCTURE ONLY (imported by tests/, __graft_entry__.smoke() and bench.py's CPU legs; never by the
product path).

CPU restatement of the reference's inference pre-processing (SURVEY.md 8(f) row f1):
  * dataset/custom_dataset.py:42-68  aug_croppad: scale = min(832/W, 512/H); cv2.resize(img, (0,0), fx=scale, fy=scale)
                                     (INTER_LINEAR on uint8 BGR); gray-128 padding left/right or top/bottom to 832x512
  * dataset/custom_dataset.py:23-24,35  torchvision ToTensor (HWC uint8 -> CHW float32 / 255) + Normalize(mean, std) with
                                     cfg.INPUT.MEANS / STDS (exps/stage3_root2/config.py:34-35)
  * exps/stage3_root2/test.py:99-103  default intrinsics appended to the scale dict when no ground truth exists

cv2.resize is a third-party dependency of the reference (opencv-python, unpinned in requirements.txt; 4.13.0 here).  Its
8-bit bilinear path is fixed point (modules/imgproc/src/resize.cpp: HResizeLinear<uchar,int,short,INTER_RESIZE_COEF_SCALE=2048>,
VResizeLinear<uchar,int,short,FixedPtCast<int,uchar,22>>): coefficients are float32 weights rounded (half to even) to
1/2048 steps, the horizontal pass keeps 32-bit sums and the vertical pass computes
((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.  An exact 1/2 scale is rerouted to INTER_AREA, i.e. the
rounded mean of each 2x2 block (of the pixels inside it where the image's last odd column or row cuts the block).  A side
that rounds to 0 pixels is refused, as cv2 refuses it.  tests/test_oracle_preprocess.py pins this restatement against cv2
itself and against digests of the reference pipeline's outputs (tests/golden/make_golden.py).
"""
import numpy as np

NET_W, NET_H = 832, 512
MEANS = np.array([0.406, 0.456, 0.485], np.float32)  # BGR, exps/stage3_root2/config.py:34
STDS = np.array([0.225, 0.224, 0.229], np.float32)   # exps/stage3_root2/config.py:35


def cv_round(v):
    """cvRound(double): round half to even."""
    return int(np.rint(v))


def linear_tables(src, dst, inv_scale):
    """resize.cpp (INTER_LINEAR, fixed point): -> (ofs int32 [dst], coef int16 [dst,2])."""
    scale = 1.0 / inv_scale
    ofs = np.zeros(dst, np.int32)
    coef = np.zeros((dst, 2), np.int16)
    for d in range(dst):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = np.float32(f - np.float32(s))
        if s < 0:
            f, s = np.float32(0), 0
        if s >= src - 1:
            f, s = np.float32(0), src - 1
        ofs[d] = s
        c0 = np.float32(1.0) - f
        coef[d, 0] = cv_round(float(np.float32(c0 * np.float32(2048))))
        coef[d, 1] = cv_round(float(np.float32(f * np.float32(2048))))
    return ofs, coef


def resize_linear_u8(img, fx):
    """cv2.resize(img, (0, 0), fx=fx, fy=fx) for uint8 HWC images.  Raises ValueError where cv2 raises (!dsize.empty()):
    a side that rounds to 0 pixels."""
    H, W = img.shape[:2]
    dw, dh = cv_round(W * fx), cv_round(H * fx)
    if dw <= 0 or dh <= 0:
        raise ValueError("a %dx%d image resizes to %dx%d at scale %r" % (W, H, dw, dh, fx))
    if (dw, dh) == (W, H):
        return img.copy()
    scale = 1.0 / fx
    if int(scale) == 2 and abs(2 - scale) < np.finfo(np.float64).eps:   # INTER_LINEAR -> INTER_AREA (fast 2x2 mean)
        # dw = rint(W / 2) rounds up when W = 3 (mod 4) (likewise H): the last column's (row's) windows are cut by the image
        # edge.  resizeAreaFast_Invoker averages the pixels inside such a window as saturate_cast<uchar>((float)sum / count),
        # i.e. the float quotient rounded half to even; full windows keep the SIMD path's (sum + 2) >> 2.
        s = img.astype(np.int32)
        acc = np.zeros((dh, dw, 3), np.int32)
        cnt = np.zeros((dh, dw, 1), np.int32)
        for oy in (0, 1):
            for ox in (0, 1):
                p = s[oy::2, ox::2][:dh, :dw]
                acc[:p.shape[0], :p.shape[1]] += p
                cnt[:p.shape[0], :p.shape[1]] += 1
        part = np.rint(acc.astype(np.float32) / cnt.astype(np.float32))
        return np.where(cnt == 4, (acc + 2) >> 2, part).astype(np.uint8)
    xo, xa = linear_tables(W, dw, fx)
    yo, yb = linear_tables(H, dh, fx)
    # the vertical taps of the generic resizer are clamped row indices around floor(fy) WITHOUT the f=0 snap used for x:
    # rows = clip(sy, 0, H-1), clip(sy+1, 0, H-1) with the unsnapped weights
    yo2 = np.zeros((dh, 2), np.int32)
    yb2 = np.zeros((dh, 2), np.int16)
    for d in range(dh):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = np.float32(f - np.float32(s))
        yo2[d] = (min(max(s, 0), H - 1), min(max(s + 1, 0), H - 1))
        yb2[d, 0] = cv_round(float(np.float32((np.float32(1.0) - f) * np.float32(2048))))
        yb2[d, 1] = cv_round(float(np.float32(f * np.float32(2048))))
    src = img.astype(np.int32)
    x1 = np.minimum(xo + 1, W - 1)
    hor = src[:, xo, :] * xa[:, 0].astype(np.int32)[None, :, None] + src[:, x1, :] * xa[:, 1].astype(np.int32)[None, :, None]
    s0 = hor[yo2[:, 0]] >> 4
    s1 = hor[yo2[:, 1]] >> 4
    b0 = yb2[:, 0].astype(np.int32)[:, None, None]
    b1 = yb2[:, 1].astype(np.int32)[:, None, None]
    out = (((b0 * s0) >> 16) + ((b1 * s1) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def aug_croppad(img):
    """dataset/custom_dataset.py:42-68 -> (uint8 [512,832,3], scale dict)."""
    H, W = img.shape[:2]
    s = min(NET_W / W, NET_H / H)
    out = resize_linear_u8(img, s)
    scale = {"scale": s, "img_width": W, "img_height": H, "net_width": NET_W, "net_height": NET_H}
    if out.shape[1] < NET_W:
        ml = (NET_W - out.shape[1]) // 2
        mr = NET_W - out.shape[1] - ml
        out = np.concatenate((np.full((out.shape[0], ml, 3), 128, np.uint8), out, np.full((out.shape[0], mr, 3), 128, np.uint8)), axis=1)
    elif out.shape[0] < NET_H:
        mu = (NET_H - out.shape[0]) // 2
        md = NET_H - out.shape[0] - mu
        out = np.concatenate((np.full((mu, out.shape[1], 3), 128, np.uint8), out, np.full((md, out.shape[1], 3), 128, np.uint8)), axis=0)
    return out, scale


def to_tensor_normalize(img_u8):
    """ToTensor + Normalize (float32): ((u8 / 255) - mean) / std, HWC -> CHW."""
    x = img_u8.astype(np.float32) / np.float32(255)
    x = (x - MEANS[None, None, :]) / STDS[None, None, :]
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def default_intrinsics(scale):
    """exps/stage3_root2/test.py:99-103 (no ground truth)."""
    s = dict(scale)
    s["f_x"] = s["img_width"]
    s["f_y"] = s["img_width"]
    s["cx"] = s["img_width"] / 2
    s["cy"] = s["img_height"] / 2
    return s


def preprocess(img):
    """uint8 BGR [H,W,3] -> (float32 [3,512,832], scale dict with intrinsics)."""
    u8, scale = aug_croppad(img)
    return to_tensor_normalize(u8), default_intrinsics(scale)
