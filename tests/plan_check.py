"""The per-op checker of the backbone plan, one for every precision (bf16x3, bf16, fp16), and what the GPU tests around
it share: plan introspection (smapb_debug_checksums, smapb_debug_dump), float64 references of one layer fed the exact
inputs the op consumed, the op loop check_ops, forced tile widths that must not change a bit, and the single-conv checker
(conv_op, check_conv: a conv_test call described as a plan op and judged by the same judge()) of
tests/test_conv_gpu.py, tests/test_fp16_gpu.py and tests/test_conv_edges_gpu.py.

The reference r of an op is computed in fp64 from the operands the device holds (folded as the library folds them), so
what separates the device from it is fp32 arithmetic: every element must lie within its precision's output rounding
plus a probabilistic accumulation bound 8 u sqrt(K + 8) (|pre| + |r| + 4 Q), u = 2^-24, Q^2 = the sum of the squared
terms (_acc_bound):
  * bf16x3: 2^-17 |r|, r built from hi + lo weights with the a_lo w_lo product the three MMAs leave out ("dev3");
    `-s` also prints the per-channel error against it and against the float64 layer of the unfolded state dict;
  * bf16: 1 ulp_bf16(r), bf16 weights;
  * fp16: 1/2 ulp_fp16(y) against clamp(r) to +-65504 (the store's clamp; on in-range data clamp(r) == r), fp16
    weights;
  * fp32 outputs (the heads), in every precision: |y| 2^-24.
Where an op ends in its ReLU and r's pre-activation is below minus its accumulation bound, the output is exactly 0;
padded channels are exactly 0; the max-pool and the space-to-depth view match bit for bit; the returned heads
(head_merge, tapsum) are within 1e-5 of max of their recomputation from the dumped fp32 heads.  The wrong references
of _MUTATIONS that apply to a plan are tried and must be flagged.

Not a test module: it makes no CUDA call at import."""
import ctypes
import math
import time

import pytest
import torch
import torch.nn.functional as F

from oracle import smap_torch

DESC_BYTES = 512
MAX_OPS = 1024
TOL_HEADS = 1e-5
FP16_MAX = 65504.0
SEED = 5
ROLES = ("in", "in2", "res", "p1", "p2", "up", "a")  # the inputs an op description may name


def no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _gid(g, width_first=False):
    """Test id of a geometry (H, W, B): "HxW_bB", or "WxH_bB"."""
    H, W, B = g
    return "%dx%d_b%d" % ((W, H, B) if width_first else (H, W, B))


# ---------------------------------------------------------------------------------------------------------------------
# plan introspection
# ---------------------------------------------------------------------------------------------------------------------
def _debug_fns(lib):
    c = ctypes
    lib.smapb_debug_checksums.argtypes = [c.c_void_p, c.c_int, c.POINTER(c.c_ulonglong), c.c_int, c.c_void_p, c.c_int]
    lib.smapb_debug_checksums.restype = c.c_int
    lib.smapb_debug_dump.argtypes = [c.c_void_p, c.c_int, c.c_int, c.c_void_p, c.c_longlong, c.c_int]
    lib.smapb_debug_dump.restype = c.c_longlong
    return lib


def plan_ops(eng, B):
    """-> (checksums, descriptions): one dict per dumped op of the batch-B plan, as left by the last forward."""
    lib = _debug_fns(eng.lib)
    sums = (ctypes.c_ulonglong * MAX_OPS)()
    buf = ctypes.create_string_buffer(MAX_OPS * DESC_BYTES)
    n = lib.smapb_debug_checksums(eng._h, B, sums, MAX_OPS, buf, DESC_BYTES)
    assert 0 < n < MAX_OPS, (n, lib.smapb_last_error(eng._h))
    ops = []
    for i in range(n):
        s = buf.raw[i * DESC_BYTES:(i + 1) * DESC_BYTES].split(b"\0", 1)[0].decode()
        d = dict(kv.split("=", 1) for kv in s.split())
        d["idx"] = i
        ops.append(d)
    return [int(v) for v in sums[:n]], ops


def _dims(op):
    return [int(v) for v in op["out"].split("x")]


def dump(eng, B, op):
    """Op output on the device: [planes, N, H, W, C] in bf16 (hi, and lo when nterms > 1) or fp16 (dtype=f16, one
    plane), or fp32 [N, H, W, C] (conv_f32)."""
    N, H, W, C = _dims(op)
    if op["kind"] == "conv_f32":
        t = torch.empty(N, H, W, C, dtype=torch.float32, device="cuda")
    elif op.get("dtype") == "f16":
        t = torch.empty(1, N, H, W, C, dtype=torch.float16, device="cuda")
    else:
        t = torch.empty(int(op["nterms"]) // 2 + 1, N, H, W, C, dtype=torch.bfloat16, device="cuda")
    nbytes = t.numel() * t.element_size()
    got = _debug_fns(eng.lib).smapb_debug_dump(eng._h, B, op["idx"], ctypes.c_void_p(t.data_ptr()), nbytes, 0)
    assert got == nbytes, (op["name"], got, nbytes)
    return t


def value(t, hi_only=False):
    """fp64 value a dumped tensor carries: the sum of its planes (exact in fp64), the fp32 output itself, or hi alone."""
    if t.dtype == torch.float32:
        return t.double()
    return t[0].double() if hi_only else t.double().sum(0)


def op_class(op):
    k = op["kind"]
    if k == "conv":
        if "in2" in op:
            return "fused_pair_s%s" % op["s2"]
        if "up" in op:
            return "up_residual"
        if "p2" in op:
            return "res_p1_p2"
        if "res" in op:
            return "residual"
        return "conv%s" % op["k"]
    if k == "conv_f32":
        return "tapexp" if op["name"].endswith(".tapexp") else "head_f32"
    return k


def _consumers(ops):
    """Producer index -> the indices of the ops that read its output."""
    uses = {}
    for op in ops:
        for r in ROLES:
            if r in op and op[r] != "x":
                uses.setdefault(int(op[r]), []).append(op["idx"])
    return uses


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------
class Weights:
    """Per-unit (W, bias, W_lo) with conv(x, W) + bias == BN_eval(conv(x, w, b)).  mode "x3": float64 from the unfolded
    state dict.  Modes "bf16", "dev3" and "fp16" hold what the device holds - folded as fold_unit does (float64, rounded
    to fp32), fused-pair biases the fp32 sum of the two folded biases - with weights rounded to bf16 ("bf16"), carried
    as hi + lo ("dev3", W = hi + lo and W_lo = lo: the bf16x3 MMAs compute a (w_hi + w_lo) - a_lo w_lo) or rounded to
    fp16 ("fp16")."""

    def __init__(self, sd, mode):
        self.sd, self.mode, self.cache = sd, mode, {}

    def unit(self, name):
        if name not in self.cache:
            g = lambda k: self.sd[name + k].double().cuda()  # noqa: E731
            w, b = g(".conv.weight"), g(".conv.bias")
            s = g(".bn.weight") / torch.sqrt(g(".bn.running_var") + smap_torch.BN_EPS)
            W = w * s.view(-1, 1, 1, 1)
            bias = (b - g(".bn.running_mean")) * s + g(".bn.bias")
            self.cache[name] = device_form(W, bias, self.mode)
        return self.cache[name]

    def bias_sum(self, b1, b2):
        return b1 + b2 if self.mode == "x3" else (b1 + b2).double()  # an fp32 add on the device


def device_form(W, bias, mode):
    """(W, bias, W_lo) of float64 weights W and bias as the device holds them in `mode` (see Weights); W is rounded to fp32
    first, as upload_conv_layer receives it.  Mode "x3": unchanged, no W_lo."""
    if mode == "x3":
        return W, bias, None
    wf, lo = W.float(), None
    if mode == "fp16":
        W = wf.half().double()
    else:
        hi = wf.bfloat16()
        W = hi.double()
        if mode == "dev3":
            lo = (wf - hi.float()).bfloat16().double()
            W = W + lo
    return W, bias.float(), lo


class ConvWeights:
    """Weights-like source of one conv_test call: its raw fp32 weights w [Cout, Cin + Cin2, k, k] and bias b, in the
    device's form (device_form; mode "dev3", "bf16" or "fp16").  A K-concatenated pair (op name ending in
    fused_conv3_downsample) is served as reference() asks for it: "<base>conv_bn_relu3" the first Cin columns with the bias,
    "<base>downsample" the other Cin2 columns with a zero bias (b + 0 is b in fp32)."""

    def __init__(self, w, b, cin, mode):
        self.mode, self.cin = mode, cin
        self.W, self.bias, self.lo = device_form(w.double(), b.double(), mode)

    def unit(self, name):
        cols = slice(None)
        bias = self.bias
        if name.endswith("conv_bn_relu3"):
            cols = slice(0, self.cin)
        elif name.endswith("downsample"):
            cols, bias = slice(self.cin, None), torch.zeros_like(bias)
        return self.W[:, cols], bias, None if self.lo is None else self.lo[:, cols]

    def bias_sum(self, b1, b2):
        return (b1 + b2).double()


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _conv(x, W, stride=1, pad=0):
    """x fp64 NHWC (channels beyond W's Cin ignored) -> fp64 NHWC, no bias."""
    return _nhwc(F.conv2d(_nchw(x[..., :W.shape[1]]), W, stride=stride, padding=pad))


def _coeff(n_in, n_out, device):
    """Bilinear align_corners=True indices and weights for one axis, computed in fp32 as ATen (and the kernels) do."""
    scale = torch.tensor(float(n_in - 1), dtype=torch.float32) / torch.tensor(float(n_out - 1), dtype=torch.float32) \
        if n_out > 1 else torch.tensor(0.0)
    src = scale * torch.arange(n_out, dtype=torch.float32)
    i0 = src.long()
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = src - i0.float()
    l0 = 1 - l1
    return i0.to(device), i1.to(device), l0.double().to(device), l1.double().to(device)


def _up(t, H, W, align_corners=True):
    """Bilinear resize of fp64 NHWC t to H x W: the exact fp64 combination with the fp32 weights of the reference
    model's F.interpolate(align_corners=True); align_corners=False only serves as a deliberately wrong reference."""
    if not align_corners:
        return _nhwc(F.interpolate(_nchw(t), size=(H, W), mode="bilinear", align_corners=False))
    y0, y1, hy0, hy1 = _coeff(t.shape[1], H, t.device)
    x0, x1, wx0, wx1 = _coeff(t.shape[2], W, t.device)
    a, b = t[:, y0], t[:, y1]
    v = lambda u: u[:, :, x0] * wx0.view(1, 1, -1, 1) + u[:, :, x1] * wx1.view(1, 1, -1, 1)  # noqa: E731
    return v(a) * hy0.view(1, -1, 1, 1) + v(b) * hy1.view(1, -1, 1, 1)


def _image_from_s2d(s2d_val, H, W):
    """Invert the space-to-depth view: [N, H/2, W/2+3, 16] -> NCHW image (channel (by*2+bx)*3+c, columns 2..W/2+1)."""
    N = s2d_val.shape[0]
    v = s2d_val[:, :, 2:2 + W // 2, :12].reshape(N, H // 2, W // 2, 2, 2, 3)  # n, y, x, by, bx, c
    return v.permute(0, 5, 1, 3, 2, 4).reshape(N, 3, H, W)


def s2d_expected(img, precision):
    """The planes the s2d kernel must write for fp32 image img [N,3,H,W]: split bf16 (hi, and lo in bf16x3), or one fp16
    plane of the documented mapping (NaN -> -65504, beyond the range -> +-65504: the identity on in-range images)."""
    N, _, H, W = img.shape
    if precision == "fp16":
        img = torch.where(torch.isnan(img), torch.full_like(img, -FP16_MAX), img).clamp(-FP16_MAX, FP16_MAX)
    v = img.reshape(N, 3, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(N, H // 2, W // 2, 12)
    v = F.pad(v, (0, 4, 2, 1))
    if precision == "fp16":
        return v.half()[None]
    hi = v.bfloat16()
    planes = [hi] if precision == "bf16" else [hi, (v - hi.float()).bfloat16()]
    return torch.stack(planes)


def reference(op, get, wts, image, mut=None, squares=False, get_lo=None):
    """fp64 reference of one op -> (r, pre, relu_last), NHWC with the layer's real channel count.  get(role) returns the
    fp64 value of an input; mut names a deliberately wrong variant; squares=True evaluates the same expression on squared
    inputs, weights and biases, without the ReLU (Q^2 of _acc_bound: the sum of the squared terms an output element
    accumulates); get_lo(role) (with "dev3" weights) returns the lo plane of an input, for the a_lo w_lo product the
    bf16x3 MMAs leave out."""
    A = (lambda t: t * t) if squares else (lambda t: t)  # noqa: E731
    name, kind = op["name"], op["kind"]

    def unit(n):
        W, b, Wlo = wts.unit(n)
        if mut == "bias_shift" and W.shape[0] >= 64:  # chunk 0's bias replaced by chunk 1's
            b = b.clone()
            b[:32] = b[32:64]
        if mut in ("drop_hi_wlo", "plain_bf16") and Wlo is not None:  # bf16x3 without its a_hi w_lo MMA
            W, Wlo = W - Wlo, None
        return A(W), A(b), Wlo

    def cv(role, W, Wlo, xform=lambda t: t, **kw):  # conv of input `role`, minus a_lo w_lo where the device drops it
        r = _conv(xform(A(get(role))), W, **kw)
        if Wlo is not None and get_lo is not None:
            r = r - _conv(xform(get_lo(role)), Wlo, **kw)
        return r

    if kind in ("stem_tc", "stem"):
        W, b, Wlo = unit("top.conv")
        if kind == "stem_tc":
            to_img = lambda t: _nhwc(_image_from_s2d(t, image.shape[2], image.shape[3]))  # noqa: E731
            pre = cv("in", W, Wlo, xform=to_img, stride=2, pad=3) + b
        else:  # the CUDA-core stem: fp32 image and fp32 weights
            if wts.mode != "x3":
                W = A(Weights(wts.sd, "x3").unit("top.conv")[0].float().double())
            pre = _conv(_nhwc(A(image.double())), W, stride=2, pad=3) + b
        return (pre if squares else F.relu(pre)), pre, True
    if kind == "conv_f32" and name.endswith(".tapexp"):
        W, _, Wlo = unit(name[:-len(".tapexp")])
        C = W.shape[0]
        expand = lambda w: w.permute(2, 3, 0, 1).reshape(9 * C, w.shape[1], 1, 1)  # noqa: E731  row (ky*3+kx)*C + c
        r = cv("in", expand(W), None if Wlo is None else expand(Wlo))
        return r, r, False
    if kind == "conv_f32":
        W, b, Wlo = unit(name)
        r = cv("in", W, Wlo, pad=int(op["pad"].split("x")[0])) + b
        return r, r, False
    assert kind == "conv", "no reference for op kind %r (%s)" % (kind, name)
    stride, pad = int(op["s"]), int(op["pad"].split("x")[0])
    def last_kb(W, Wlo):  # the weights of the conv's last k-block (tap ky = kh-1, kx = kw-1, last 64 channels) zeroed
        if mut != "drop_last_kb":
            return W, Wlo
        W = W.clone()
        W[:, -64:, -1, -1] = 0
        if Wlo is not None:
            Wlo = Wlo.clone()
            Wlo[:, -64:, -1, -1] = 0
        return W, Wlo

    if "in2" in op:  # relu(conv3(o2) + downsample(t)) as one K-concatenated GEMM
        base = name[:-len("fused_conv3_downsample")]
        W3, b3, W3lo = unit(base + "conv_bn_relu3")
        Wd, bd, Wdlo = unit(base + "downsample")
        Wd, Wdlo = last_kb(Wd, Wdlo)  # the second input's k-blocks come last
        shift = (lambda t: torch.roll(t, 1, dims=2)) if mut == "shift_ds" else (lambda t: t)
        pre = cv("in", W3, W3lo) + cv("in2", Wd, Wdlo, xform=shift, stride=int(op["s2"])) + wts.bias_sum(b3, bd)
    else:
        W, b, Wlo = unit(name)
        W, Wlo = last_kb(W, Wlo)
        pre = cv("in", W, Wlo, stride=stride, pad=pad) + b
    C = pre.shape[-1]
    if "res" in op:
        pre = pre + A(get("res"))[..., :C]
    if "up" in op:
        pre = pre + _up(A(get("up"))[..., :C], pre.shape[1], pre.shape[2], mut != "align_false")
    r = F.relu(pre) if int(op["relu"]) and not squares else pre
    posts = [p for p in ("p1", "p2") if p in op]
    if mut == "drop_post2":
        posts = posts[:1]
    for p in posts:
        r = r + A(get(p))[..., :C]
    return r, pre, int(op["relu"]) == 1 and "p1" not in op


def x3_error(y, r, pre, relu_last, neg=None):
    """-> (worst per-channel normalised error, list of violated exact conditions).  Where the reference pre-activation of
    an op that ends in its ReLU is below -neg (default 1e-6 max|r|), the output must be exactly 0."""
    C = r.shape[-1]
    assert y.shape[:-1] == r.shape[:-1] and y.shape[-1] >= C, (tuple(y.shape), tuple(r.shape))
    rmax = r.abs().max()
    den = torch.clamp(r.abs().amax(dim=(0, 1, 2)), min=1e-3 * rmax.item())
    err = ((y[..., :C] - r).abs().amax(dim=(0, 1, 2)) / den).max().item()
    bad = []
    if relu_last and ((pre < -(1e-6 * rmax if neg is None else neg)) & (y[..., :C] != 0)).any():
        bad.append("non-zero output where the pre-activation is negative")
    if y.shape[-1] > C and (y[..., C:] != 0).any():
        bad.append("padded channels not zero")
    return err, bad


def _ulp_bf16(r):
    _, e = torch.frexp(r)  # |r| = m 2^e, m in [0.5, 1): ulp = 2^(e - 1 - 7)
    return torch.where(r != 0, torch.ldexp(torch.ones_like(r), e - 8), torch.zeros_like(r))


def half_ulp16(y):
    """Half an fp16 ulp of fp16 values y (fp64 tensor): the round-to-nearest error of the store that produced them."""
    a = y.abs()
    _, e = torch.frexp(a)  # a = m 2^e, m in [0.5, 1): ulp = 2^(e - 1 - 10), subnormal ulp 2^-24
    e = torch.clamp(e - 11, min=-24)
    return torch.ldexp(torch.full_like(a, 0.5), e)


def _K(op):
    """Products one output element accumulates.  The CUDA-core stem: 7x7x3 fp32 FMAs (then the bias, one of the 8
    roundings _acc_bound adds)."""
    if op["kind"] == "stem":
        return 147
    kh, kw = (int(v) for v in op.get("k", "1x1").split("x"))
    return kh * kw * int(op.get("cin", 0)) + int(op.get("cin2", 0))


LAMBDA = 8.0  # tail parameter of the accumulation bound: P(one element exceeds it | model) <= 2 exp(-LAMBDA^2 / 2) ~ 3e-14


def _acc_bound(op, q, *mags):
    """fp32 arithmetic bound of one output element.  The reference uses the device's own operands (bf16 or fp16 weights
    in the one-MMA precisions; hi + lo weights and the dropped a_lo w_lo product in bf16x3; fp32 folded biases) and
    products of bf16 or fp16 values are exact, so what separates the device from it is fp32 accumulation (plus the
    output rounding, added by the caller).
    To first order that error is sum_k d_k S_k over the n = K + 8 roundings of the element (K products, bias, residual
    or the ~6 roundings of the bilinear term, two skips), with |d_k| <= u = 2^-24 and S_k the running sum.  With the
    rounding errors modelled as independent and mean-zero (Higham & Mary, "A new approach to probabilistic rounding error
    analysis", 2019), Hoeffding's inequality gives |error| <= LAMBDA u sqrt(sum_k S_k^2) <= LAMBDA u sqrt(n) max_k |S_k|
    except with probability 2 exp(-LAMBDA^2 / 2).  A running sum of terms t_i is the final value's share plus a bridge
    whose spread is set by Q = sqrt(sum t_i^2); max_k |S_k| <= |pre| + |r| + 4 Q covers it (4 standard deviations of
    the bridge, with pre and r the sums before and after the ReLU and skips).  Unlike the worst case n u sum |t_i|, this
    grows like sqrt(K) Q, so it separates bf16x3 (fp32-faithful products) from any bf16-level product error
    (~2^-9 Q) at every K of the network: the checker is shown to flag hi-only activations, a dropped a_hi w_lo MMA and
    plain-bf16 products on the largest-K conv of each geometry."""
    m = 4 * q
    for t in mags:
        m = m + t.abs()
    return LAMBDA * 2.0 ** -24 * math.sqrt(_K(op) + 8) * m


def split3(r, b):
    """-> (sure-over, sure-in, band) masks of reference values r with accumulation bound b."""
    a = r.abs()
    over = a - b > FP16_MAX
    inside = a + b <= FP16_MAX
    return over, inside, ~(over | inside)


def clamp_check(y, r, b):
    """fp16 outputs y (fp64, real channels) against r: -> (sure-over mask, band mask, worst |y - clamp(r)| / bound,
    violated conditions)."""
    over, _, band = split3(r, b)
    bad = []
    if not torch.equal(y[over], torch.sign(r[over]) * FP16_MAX):
        bad.append("%d sure-over elements not stored as +-65504" % int((y[over].abs() != FP16_MAX).sum().item()))
    bound = half_ulp16(y) + b
    err = ((y - r.clamp(-FP16_MAX, FP16_MAX)).abs() / bound.clamp(min=1e-30)).max().item()
    if err > 1.0:
        bad.append("error %.3g x the bound" % err)
    return over, band, err, bad


# ---------------------------------------------------------------------------------------------------------------------
# per-op parity of one plan
# ---------------------------------------------------------------------------------------------------------------------
_MUTATIONS = {  # deliberately wrong reference -> op classes it applies to (largest_k: the conv with the most products)
    "align_false": ("up_residual",),
    "drop_post2": ("res_p1_p2",),
    "shift_ds": ("fused_pair_s2",),
    "bias_shift": ("conv1x1",),
    "hi_only": ("largest_k",),      # bf16x3 with the activations' lo plane dropped
    "drop_hi_wlo": ("largest_k",),  # bf16x3 without the a_hi w_lo MMA
    "plain_bf16": ("largest_k",),   # a_hi w_hi only
}  # and, for single convs only (conv_mutations), "drop_last_kb": without the last k-block (last tap, last 64 channels)
_X3_ONLY = ("hi_only", "drop_hi_wlo", "plain_bf16")


def applicable_mutations(ops, precision):
    """The wrong references check_ops must flag on a plan: those whose op class occurs in it."""
    classes = {op_class(o) for o in ops} | {"largest_k"}
    return {m for m, cls in _MUTATIONS.items()
            if classes & set(cls) and not (m in _X3_ONLY and precision != "bf16x3")}


def _changes(rm, r):
    """Whether a wrong reference differs from the right one by more than fp64 rounding (it may not: bilinear
    interpolation from a 1-pixel level is the same with and without align_corners, a bias chunk may equal the next)."""
    return (rm - r).abs().max().item() > 1e-12 * r.abs().max().item()


def f32_out(op):
    """Whether a conv stores fp32 (the heads, or a conv_test call with an fp32 output) rather than activation planes."""
    return op["kind"] == "conv_f32" or op.get("f32") == "1"


def out_rounding(op, precision, yc):
    """The output-rounding term of an element's bound, as a function of the reference r: fp32 outputs |y| 2^-24 (one
    fp32 rounding, in every precision); bf16x3 2^-17 |r| (hi + lo carries the fp32 value to 2^-18 relative); bf16 1 ulp
    of r (<= 1/2 ulp of the fp32 value, <= 1 ulp(r) within a binade of r); fp16 1/2 ulp of the stored y."""
    if f32_out(op):
        return lambda r: yc.abs() * 2.0 ** -24
    if precision == "bf16x3":
        return lambda r: 2.0 ** -17 * r.abs() * (1 + 2.0 ** -20)
    if precision == "bf16":
        return lambda r: _ulp_bf16(r) * (1 + 2.0 ** -20)
    return lambda r: half_ulp16(yc)


def judge(op, y, get, rw, precision, img=None, get_lo=None, muts=()):
    """One conv-like op's output y (fp64 NHWC, padded channels after the real ones) against the float64 reference of the
    device's operands (weights rw; inputs get(role, hi_only), lo planes get_lo(role) in bf16x3): every element within
    out_rounding + _acc_bound, exact zeros where the ReLU must clear, padded channels zero, and in fp16 the store's clamp
    (clamp_check).  Each wrong reference of muts (keys of _MUTATIONS, or "drop_last_kb") is compared with y by the same
    bound.
    -> dict r, pre (the right reference), err (worst |y - r| / bound), share (of the elements outside the bound), bad
    (violated conditions), over and band (fp16 stores: sure-over and band masks, else None) and tried: wrong reference -> (flagged, share of the elements outside the
    bound), without those that equal the right reference here (_changes)."""
    r, pre, relu_last = reference(op, get, rw, img, get_lo=get_lo)
    q = reference(op, get, rw, img, squares=True)[0].sqrt()
    yc = y[..., :r.shape[-1]]
    clamp = precision == "fp16" and not f32_out(op)  # fp16 stores clamp to +-65504; fp32 outputs do not
    out_round = out_rounding(op, precision, yc)

    def bound(r, pre):
        return out_round(r) + _acc_bound(op, q, r, pre)

    def dist(r):
        return (yc - (r.clamp(-FP16_MAX, FP16_MAX) if clamp else r)).abs()

    # exact zeros where the ReLU must clear (pre below minus its own accumulation bound), padded channels
    bad = x3_error(y, r, pre, relu_last, neg=_acc_bound(op, q, pre))[1]
    out = {"r": r, "pre": pre, "over": None, "band": None, "tried": {}}
    if clamp:
        if not torch.isfinite(y).all():
            bad.append("non-finite activations")
        over, in_band, err, more = clamp_check(yc, r, _acc_bound(op, q, r, pre))
        bad += more
        out.update(over=over, band=in_band)
    else:
        err = (dist(r) / bound(r, pre).clamp(min=1e-30)).max().item()
        if err > 1.0:
            bad.append("error %.3g x the bound" % err)
    out["share"] = (dist(r) > bound(r, pre)).double().mean().item()
    # the wrong references (host-side only: the same device output)
    for mut in muts:
        hi = mut in ("hi_only", "plain_bf16")
        rm, pm, _ = reference(op, lambda role: get(role, hi), rw, img, mut=mut,
                              get_lo=None if hi or precision != "bf16x3" else get_lo)
        if not _changes(rm, r):
            continue
        over = dist(rm) > bound(rm, pm)
        zeros = bool(x3_error(y, rm, pm, relu_last, neg=_acc_bound(op, q, pm))[1])
        out["tried"][mut] = (bool(over.any()) or zeros, over.double().mean().item())
    out.update(err=err, bad=bad)
    return out


def check_ops(eng, B, sd, img, outs, precision):
    """Every dumped op of the batch-B plan, as left by the last forward (of img, which returned outs), against its
    float64 reference, and the returned heads against the dumped head outputs.  Each wrong reference is tried on the
    first op of its class where it differs from the right one.  -> summary dict:
      ops, failures       the op descriptions, one line per op that broke a condition;
      worst               worst |y - r| / bound per op class (heads: error / max);
      flagged             wrong reference -> whether the checker rejected it;
      per_channel         bf16x3: op class -> worst per-channel error against the device-operand and the unfolded
                          float64 reference (printed, not asserted);
      over, neg, band     fp16: sure-over elements per op class, those of them below -65504, band elements;
      lo, hi              fp16: the interval [sum sure-over, sum sure-over + band] a saturation count must lie in."""
    fp16 = precision == "fp16"
    _, ops = plan_ops(eng, B)
    wts = Weights(sd, {"bf16x3": "x3", "bf16": "bf16", "fp16": "fp16"}[precision])
    rw = Weights(sd, "dev3") if precision == "bf16x3" else wts  # the operands the device holds
    uses = _consumers(ops)
    live, heads = {}, {}
    worst, per_channel, flagged, failures = {}, {}, {}, []
    over_by, band, neg = {}, 0, 0
    largest_k = max((o for o in ops if o["kind"] == "conv"), key=_K)["idx"]
    for op in ops:
        i, cls = op["idx"], op_class(op)
        bad, err, n_over = [], 0.0, 0
        if fp16 and op["kind"] != "conv_f32" and op.get("dtype") != "f16":
            bad.append("description lacks dtype=f16")
        y_raw = dump(eng, B, op)
        if uses.get(i):
            live[i] = y_raw  # kept until its last consumer is checked

        def get(role, hi_only=False):
            return value(live[int(op[role])], hi_only)

        def get_lo(role):
            return live[int(op[role])][1].double()

        if op["kind"] == "s2d":
            if not torch.equal(y_raw, s2d_expected(img, precision)):
                err = math.inf
                bad.append("s2d planes differ")
            if fp16:
                n_over = int((~(img.abs() <= FP16_MAX)).sum().item())
        elif op["kind"] == "maxpool":
            if not torch.equal(value(y_raw), _nhwc(F.max_pool2d(_nchw(get("a")), 3, 2, 1))):
                err = math.inf
                bad.append("max-pool not bit-exact")
        else:
            y = value(y_raw)
            # the checker must flag deliberately wrong references: those not yet flagged that apply to this op
            muts = [m for m, mcls in _MUTATIONS.items()
                    if m not in flagged and not (m in _X3_ONLY and precision != "bf16x3")
                    and (cls in mcls or (i == largest_k and "largest_k" in mcls))]
            j = judge(op, y, get, rw, precision, img, get_lo=get_lo, muts=muts)
            err, r, pre = j["err"], j["r"], j["pre"]
            bad += j["bad"]
            if precision == "bf16x3":
                rs, ps, relu_last = reference(op, get, wts, img)
                d0, s0 = per_channel.get(cls, (0.0, 0.0))
                per_channel[cls] = (max(d0, x3_error(y, r, pre, relu_last)[0]), max(s0, x3_error(y, rs, ps, relu_last)[0]))
            if j["over"] is not None:
                n_over = int(j["over"].sum().item())
                neg += int((j["over"] & (r < 0)).sum().item())
                band += int(j["band"].sum().item())
            for mut in muts:
                if mut not in j["tried"]:
                    print("  wrong reference %-12s on op %d %s: equals the right one here, tried on a later op"
                          % (mut, i, op["name"]))
                    continue
                flagged[mut], share = j["tried"][mut]
                print("  wrong reference %-12s on op %d %s (K %d): %.3g of its elements outside the bound"
                      % (mut, i, op["name"], _K(op), share))
        if op["kind"] == "conv_f32":
            heads[op["name"]] = y_raw
        if n_over:
            over_by[cls] = over_by.get(cls, 0) + n_over
        worst[cls] = max(worst.get(cls, 0.0), err)
        if bad:
            failures.append("op %d %s (%s, bn %s, tw %s): %s" % (i, op["name"], cls, op.get("bn"), op.get("tw"),
                                                                "; ".join(bad)))
        for j in [int(op[r]) for r in ROLES if r in op and op[r] != "x"]:
            uses[j].remove(i)
            if not uses[j]:
                live.pop(j, None)
    # the returned heads from the dumped head outputs: head_merge (upsample + sum) and tapsum (bias + taps)
    hm, dd, rd = (o.double() for o in outs)
    p = "stage2.upsample.up%d."
    r4, r3, r2 = (value(heads[(p % u) + "res_conv2"]) for u in (4, 3, 2))
    h, w = r4.shape[1], r4.shape[2]
    hm_ref = _nchw(r4 + _up(r3, h, w) + _up(r2, h, w))[:, :43]
    errs = {"head_merge": ((hm - hm_ref).abs().max() / hm_ref.abs().max()).item()}
    for key, got, C in (("res_d_conv2", dd, 14), ("res_rd_conv2", rd, 1)):
        T = F.pad(_nchw(value(heads[(p % 4) + key + ".tapexp"])), (1, 1, 1, 1))
        ref = rw.unit((p % 4) + key)[1].double().view(1, -1, 1, 1)  # the fp32 bias tapsum adds
        for t in range(9):
            ky, kx = divmod(t, 3)
            ref = ref + T[:, t * C:(t + 1) * C, ky:ky + h, kx:kx + w]
        errs["tapsum." + key] = ((got - ref).abs().max() / ref.abs().max()).item()
    for k, e in errs.items():
        worst[k] = e
        if not e <= TOL_HEADS:
            failures.append("%s: error %.3g of max > %g" % (k, e, TOL_HEADS))
    s = {"ops": ops, "worst": worst, "flagged": flagged, "failures": failures, "per_channel": per_channel}
    if fp16:
        lo = sum(over_by.values())
        s.update(over=over_by, neg=neg, band=band, lo=lo, hi=lo + band)
    return s


def check_plan(precision, H, W, B, eng=None, sd=None):
    """Run the plan twice (different images: a tile a kernel skipped keeps the first run's data), then check_ops on the
    second run; prints the worst error per op class.  The summary adds "count", the handle's saturation count after
    the two forwards.  eng: an existing handle (max_batch >= B, the state dict loaded in `precision`), left open; by
    default a handle with max_batch == B is created and closed.  sd: the state dict (default
    make_state_dict(SEED, "random"))."""
    from smap_b200.engine import Engine

    no_tf32()
    t0 = time.time()
    print("\n[plan ops %s %dx%d B=%d%s]" % (precision, H, W, B, "" if eng is None else " max_batch=%d" % eng.max_batch))
    if sd is None:
        sd = smap_torch.make_state_dict(SEED, "random")
    own = eng is None
    if own:
        eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        if own:
            eng.load_state_dict(sd, precision)
        eng.forward(smap_torch.make_input(B, H, W, seed=SEED + 1).cuda())
        img = smap_torch.make_input(B, H, W, seed=SEED + 2).cuda()
        outs = eng.forward(img)
        torch.cuda.synchronize()
        s = check_ops(eng, B, sd, img, outs, precision)
        s["count"] = eng.saturation_count()
    finally:
        if own:
            eng.close()
    torch.cuda.empty_cache()
    print("  %d ops, %.1f s; worst per op kind: |y - r| / bound (heads: error / max), and for bf16x3 the per-channel"
          " normalised error against the device-operand and the unfolded fp64 reference" % (len(s["ops"]), time.time() - t0))
    for k in sorted(s["worst"]):
        extra = "  per-channel %.3g / %.3g" % s["per_channel"][k] if k in s["per_channel"] else ""
        print("  %-22s %.3g%s" % (k, s["worst"][k], extra))
    return s


_SUMMARIES = {}


def plan_summary(precision, geom, env=None):
    """check_plan(precision, *geom), with the environment variable env = (name, value) set if given (plan options are
    read at plan build), run once per session: the tests that read one plan's check share it, and an exception it
    raised is raised again for each of them."""
    key = (precision, geom, env)
    if key not in _SUMMARIES:
        try:
            with pytest.MonkeyPatch.context() as m:
                if env:
                    m.setenv(*env)
                _SUMMARIES[key] = check_plan(precision, *geom)
        except Exception as e:  # noqa: BLE001 - re-raised for every test that reads this check
            _SUMMARIES[key] = e
    s = _SUMMARIES[key]
    if isinstance(s, Exception):
        raise s
    return s


def assert_checked(s, precision):
    """No failure, and every wrong reference that applies to the plan tried and flagged; in fp16 also no element near
    the range (no sure-over element, no band) and a device count of 0."""
    assert not s["failures"], "\n".join(s["failures"])
    want = applicable_mutations(s["ops"], precision)
    assert set(s["flagged"]) == want, "wrong references never tried: %s" % sorted(want - set(s["flagged"]))
    missed = sorted(m for m, f in s["flagged"].items() if not f)
    assert not missed, "wrong references the checker accepted: %s" % missed
    if precision == "fp16":
        assert s["lo"] == s["hi"] == 0, "sure-over %d, band %d" % (s["lo"], s["band"])
        assert s["count"] == 0, s["count"]


# ---------------------------------------------------------------------------------------------------------------------
# forced tile widths do not change the bits
# ---------------------------------------------------------------------------------------------------------------------
def run_sums(H, W, B, sd, x, precision):
    from smap_b200.engine import Engine

    eng = Engine(0, max_batch=B, in_h=H, in_w=W)
    try:
        eng.load_state_dict(sd, precision)
        outs = [o.cpu() for o in eng.forward(x)]
        torch.cuda.synchronize()
        sums, ops = plan_ops(eng, B)
    finally:
        eng.close()
    return sums, ops, outs


def check_switches(geom, monkeypatch, precision):
    """Every forced tile width (tile table rewritten, autotuner off) gives every op of the plan at geometry (H, W, B) in
    `precision` the bits of the default plan.  (Switches held in function-local statics, SMAPB_NO_GRAPH /
    SMAPB_DEBUG_STOP, cannot be toggled in one process.)"""
    from smap_b200 import _lib
    from smap_b200.engine import get_tile_table

    H, W, B = geom
    sd = smap_torch.make_state_dict(SEED, "random")
    x = smap_torch.make_input(B, H, W, seed=SEED + 3).cuda()
    base_sums, base_ops, base_outs = run_sums(H, W, B, sd, x, precision)

    def same(tag, sums, ops, outs):
        assert [o["name"] for o in ops] == [o["name"] for o in base_ops], tag
        diff = [o["name"] for o, a, b in zip(ops, sums, base_sums) if a != b]
        assert not diff, "%s: %d ops differ from the default plan, first %s" % (tag, len(diff), diff[:3])
        for a, b in zip(outs, base_outs):
            assert torch.equal(a, b), tag

    lib = _lib.load()
    table = get_tile_table()
    changed = set()
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
                sums, ops, outs = run_sums(H, W, B, sd, x, precision)
            for o, b in zip(ops, base_ops):
                if "bn" in o and o["bn"] != b["bn"]:
                    changed.add(op_class(o))
            same("SMAPB_FORCE_TILE=%d" % bn, sums, ops, outs)
    finally:
        lib.smapb_set_tile_table(table.encode())
    assert "up_residual" in changed and changed & {"fused_pair_s1", "fused_pair_s2"}, changed


# ---------------------------------------------------------------------------------------------------------------------
# single convolutions (conv_test)
# ---------------------------------------------------------------------------------------------------------------------
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

# B, H, W, Cin, Cout, k, stride, res (ReLU on): convs every tile width must give the same bits
_TILE_CASES = [(8, 32, 52, 256, 256, 3, 1, False), (8, 32, 52, 1024, 256, 1, 1, False), (2, 16, 26, 512, 512, 3, 2, False),
               (4, 64, 104, 128, 512, 1, 1, True), (2, 128, 208, 256, 64, 1, 1, False)]

CONV_MODES = {"bf16x3": "dev3", "bf16": "bf16", "fp16": "fp16"}  # precision -> the device's weight form (ConvWeights)


def conv_op(B, H, W, cin, cout, k=1, s=1, relu=True, res=False, posts=0, cin2=0, s2=1, up=False, f32=False):
    """A conv_test call described as a plan op (kind conv, the fields and roles check_ops reads), so that reference(),
    _acc_bound and judge() check it as they check the plan's ops.  The input x is [B, H, W, cin], padding k // 2; res,
    posts (1: p1, 2: p1 and p2) and up add epilogue inputs; cin2 > 0 adds a K-concatenated second input of
    ((Ho - 1) s2 + 1) x ((Wo - 1) s2 + 1) pixels (the smallest, so odd for s2 = 2) and needs k = s = 1; f32: fp32 output."""
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    op = {"name": "conv_test.fused_conv3_downsample" if cin2 else "conv_test", "kind": "conv", "k": "%dx%d" % (k, k),
          "cin": str(cin), "cin2": str(cin2), "s": str(s), "s2": str(s2), "pad": "%dx%d" % (p, p), "relu": str(int(relu)),
          "cout": str(cout), "in": "in", "geom": "%dx%dx%d" % (B, H, W), "out": "%dx%dx%dx%d" % (B, Ho, Wo, cout)}
    for role, on in (("res", res), ("p1", posts >= 1), ("p2", posts >= 2), ("in2", cin2 > 0), ("up", up)):
        if on:
            op[role] = role
    if f32:
        op["f32"] = "1"
    return op


def legacy_op(case):
    """conv_op of a case of CASES (B, H, W, Cin, Cout, k, stride, relu, res) or _TILE_CASES (..., stride, res; ReLU)."""
    B, H, W, cin, cout, k, s = case[:7]
    return conv_op(B, H, W, cin, cout, k, s, relu=case[7] if len(case) == 9 else True, res=case[-1])


def conv_inputs(op, seed, device="cuda"):
    """fp32 tensors of a conv_op: role -> NHWC tensor (in, and res, p1, p2, in2, up as the op names them), "w" [Cout,
    Cin + Cin2, k, k] scaled by 1 / sqrt(K) and "b" [Cout]; standard normal otherwise, so every value is in fp16's range."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    B, H, W = (int(v) for v in op["geom"].split("x"))
    _, Ho, Wo, cout = _dims(op)
    cin, cin2, k, s2 = int(op["cin"]), int(op["cin2"]), int(op["k"].split("x")[0]), int(op["s2"])
    shapes = {"in": (B, H, W, cin), "res": (B, Ho, Wo, cout), "p1": (B, Ho, Wo, cout), "p2": (B, Ho, Wo, cout),
              "in2": (B, (Ho - 1) * s2 + 1, (Wo - 1) * s2 + 1, cin2), "up": (B, Ho // 2, Wo // 2, cout)}
    t = {r: torch.randn(*shape, generator=g) for r, shape in shapes.items() if r in op}
    t["w"] = torch.randn(cout, cin + cin2, k, k, generator=g) / _K(op) ** 0.5
    t["b"] = torch.randn(cout, generator=g)
    return {r: v.to(device) for r, v in t.items()}


def run_conv(eng, op, t, precision, launch=None):
    """The device output of a conv_op on inputs t (conv_inputs): fp32 NHWC [B, Ho, Wo, Cout]."""
    return eng.conv_test(t["in"], t["w"], t["b"], res=t.get("res"), stride=int(op["s"]), relu=op["relu"] == "1",
                         precision=precision, post1=t.get("p1"), post2=t.get("p2"), in2=t.get("in2"), stride2=int(op["s2"]),
                         up=t.get("up"), out_f32=f32_out(op), launch=launch)


def device_planes(t, precision):
    """[planes, ...] of fp32 tensor t as launch_f32_to_split stores it: bf16 hi (and lo = bf16(t - hi) in bf16x3), or one
    fp16 plane."""
    if precision == "fp16":
        return t.half()[None]
    hi = t.bfloat16()
    return torch.stack([hi, (t - hi.float()).bfloat16()]) if precision == "bf16x3" else hi[None]


def conv_operands(op, t, precision):
    """-> (get, get_lo, weights) for reference() and judge(): the fp64 values of t's tensors in the planes
    launch_f32_to_split makes (device_planes), their lo planes (bf16x3), and the weights in the device's form."""
    planes = {r: device_planes(v, precision) for r, v in t.items() if r in ROLES}
    return (lambda role, hi_only=False: value(planes[role], hi_only), lambda role: planes[role][1].double(),
            ConvWeights(t["w"], t["b"], int(op["cin"]), CONV_MODES[precision]))


def check_conv(op, y, t, precision, muts=(), operands=None):
    """judge() of a conv_test output y (fp32 NHWC, real channels) against the float64 reference of the operands the device
    held (conv_operands).  operands: the precision whose operand rounding the reference assumes (default `precision`;
    another one makes a deliberately wrong reference).  -> judge's dict."""
    get, get_lo, rw = conv_operands(op, t, operands or precision)
    return judge(op, y.double(), get, rw, precision, get_lo=get_lo, muts=muts)


def conv_mutations(op, precision):
    """The wrong references that apply to a conv_op: the reference without its last k-block, a shifted bias
    chunk (Cout >= 64), hi-only activations, no a_hi w_lo MMA and plain bf16 products (bf16x3), and the one of its
    epilogue form (align_false: up; shift_ds: in2; drop_post2: p2)."""
    muts = ["drop_last_kb"] + (["bias_shift"] if int(op["cout"]) >= 64 else [])
    muts += list(_X3_ONLY) if precision == "bf16x3" else []
    return muts + [m for m, role in (("align_false", "up"), ("shift_ds", "in2"), ("drop_post2", "p2")) if role in op]
