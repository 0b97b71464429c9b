"""The float64 reference and per-element bound shared by the convolution tests that go through yb_conv2d_ex.

Every element is judged against K * unit * scale, scale = conv(|x|, |w|) + |bias| + |residual| (the magnitude its
rounding error is proportional to), never against the tensor's range.  The reference is float64 F.conv2d on the CPU;
for the fp16 modes on the fp16-rounded x, w and residual, which the kernels consume.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.error_bounds import UNIT as _UNIT, worst
from yolact_b200 import _lib

PRECISION = {"f32": 0, "f16tc": 1, "f16": 2, "f16x3": 3}     # yb_conv2d's precision argument
UNIT = dict(_UNIT, f16=_UNIT["f16tc"])
# f16tc / f16: the fp16 rounding of the output (|y| <= scale: 1 unit) + fp32 accumulation of exact fp16 products
#              (random-signed, a small fraction of a unit).
# f16x3:       hi+lo encodings of x, w and the output (1 unit each) + the dropped lo*lo product + fp32 accumulation.
# f32:         sequential fp32 accumulation, random-signed (as tests/test_gpu_dcn_edges.py).
K_BOUND = {"f16tc": 2.0, "f16": 2.0, "f16x3": 4.0, "f32": 8.0}
ACT_NONE, ACT_RELU, ACT_TANH, ACT_LEAKY = 0, 1, 2, 3
ROUNDED = ("f16tc", "f16")          # modes that consume fp16-rounded operands

RATIOS = {}   # precision -> largest err / (unit * scale) seen by the running test module

GUARD_BYTES = 4096      # on each side of a guarded output
GUARD_FILL = 0x5A       # a byte pattern unlike the 0xff poison of the output itself


@pytest.fixture(scope="module")
def hd():
    lib = _lib.load()
    yc = _lib.YbConfig()
    yc.backbone = _lib.YB_BACKBONE_NONE
    yc.num_classes, yc.mask_dim, yc.precision = 81, 32, _lib.YB_PREC_F32
    yc.nms_top_k, yc.nms_conf_thresh, yc.nms_thresh, yc.max_num_detections = 200, 0.05, 0.5, 100
    h = ctypes.c_void_p()
    _lib.check(lib.yb_create(ctypes.byref(yc), 0, ctypes.byref(h)), "yb_create")
    yield lib, h
    lib.yb_destroy(h)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    RATIOS.clear()
    yield
    for prec in sorted(RATIOS):
        print("largest err / (unit * scale), %s: %.3f" % (prec, RATIOS[prec]))


def set_mode(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def out_hw(H, W, k, stride, pad):
    return (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1


def out_shape(x, w, stride, pad, precision, o):
    """(shape, dtype) of yb_conv2d_ex's raw NHWC output for these options."""
    B, _, H, W = x.shape
    Co, _, kh, _ = w.shape
    Ho, Wo = out_hw(H, W, kh, stride, pad)
    Cp = max(Co, o.cout_pad)
    if precision == "f32" or o.y_f32:
        return (B, Ho, Wo, o.y_pix_stride or Cp), torch.float32
    return (B, Ho, Wo, (2 if precision == "f16x3" else 1) * Cp), torch.float16


def conv_ex(hd, x, w, bias, res, stride, pad, act, precision, opts=None, y=None):
    """yb_conv2d_ex with the output buffer filled with NaN first; x [B, CiP, H, W] and res are numpy fp32 NCHW, w and
    bias numpy fp32 (host).  Returns the raw output: NHWC fp32 [.., ps], fp16 [.., Cp] or hi|lo pairs [.., 2 Cp].
    y: the output tensor to write (default: a fresh one)."""
    lib, h = hd
    o = opts if opts is not None else _lib.YbConvOpts()
    o.poison = 1
    if y is None:
        shape, dtype = out_shape(x, w, stride, pad, precision, o)
        y = torch.empty(shape, device="cuda", dtype=dtype)
    B, _, H, W = x.shape
    Co, Ci, kh, kw = w.shape
    wc = np.ascontiguousarray(w, np.float32)
    bc = None if bias is None else np.ascontiguousarray(bias, np.float32)
    xd = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    rd = None if res is None else torch.from_numpy(np.ascontiguousarray(res, np.float32)).cuda()
    _lib.check(lib.yb_conv2d_ex(h, _lib.ptr(xd), wc.ctypes.data_as(ctypes.c_void_p),
                                None if bc is None else bc.ctypes.data_as(ctypes.c_void_p), _lib.ptr(rd),
                                _lib.ptr(None if o.nseg else y), B, Ci, H, W, Co, kh, kw, stride, pad, act,
                                PRECISION[precision], ctypes.byref(o), _lib.current_stream()), "yb_conv2d_ex")
    torch.cuda.synchronize()
    return y


def conv_ex_guarded(hd, x, w, bias, res, stride, pad, act, precision, opts=None):
    """conv_ex into a 16-byte aligned view inside a larger device buffer whose GUARD_BYTES on either side hold
    GUARD_FILL bytes; both bands must come back bitwise unchanged (no store outside the output tensor)."""
    o = opts if opts is not None else _lib.YbConvOpts()
    shape, dtype = out_shape(x, w, stride, pad, precision, o)
    nbytes = int(np.prod(shape)) * (4 if dtype == torch.float32 else 2)
    buf = torch.full((GUARD_BYTES + nbytes + GUARD_BYTES,), GUARD_FILL, dtype=torch.uint8, device="cuda")
    assert buf.data_ptr() % 16 == 0
    y = buf[GUARD_BYTES:GUARD_BYTES + nbytes].view(dtype).view(shape)
    conv_ex(hd, x, w, bias, res, stride, pad, act, precision, o, y=y)
    before, after = buf[:GUARD_BYTES], buf[GUARD_BYTES + nbytes:]
    for name, band in (("before", before), ("after", after)):
        changed = int((band != GUARD_FILL).sum().item())
        assert changed == 0, "%d guard bytes %s the output were overwritten" % (changed, name)
    return y


def decode(y, precision, Cp):
    """The raw NHWC output as float64 values [.., Cp]; a split pair is hi + lo * 2^-11 (common.cuh split_f32)."""
    if precision == "f16x3" and y.dtype == torch.float16:
        y = y.cpu().numpy().astype(np.float64)
        return y[..., :Cp] + y[..., Cp:] * 2.0 ** -11
    return y.cpu().numpy().astype(np.float64)[..., :Cp]


def act_f64(y, act):
    if act == ACT_RELU:
        return np.maximum(y, 0)
    if act == ACT_LEAKY:
        return np.where(y > 0, y, 0.1 * y)
    if act == ACT_TANH:
        return np.tanh(y)
    return y


def f16(a):
    return None if a is None else a.astype(np.float16).astype(np.float32)


def conv_f64(x, w, bias, stride, pad):
    """float64 conv and its magnitude conv(|x|, |w|) + |bias|, NHWC numpy."""
    xd, wd = torch.from_numpy(x).double(), torch.from_numpy(w).double()
    bd = None if bias is None else torch.from_numpy(bias).double()
    y = F.conv2d(xd, wd, bd, stride=stride, padding=pad)
    s = F.conv2d(xd.abs(), wd.abs(), None if bd is None else bd.abs(), stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).numpy(), s.permute(0, 2, 3, 1).numpy()


def check(y, ref, scale, precision, what):
    assert y.shape == ref.shape, (y.shape, ref.shape)
    err = np.abs(y - ref)
    tol = K_BOUND[precision] * UNIT[precision] * scale
    if precision in ROUNDED:
        tol = tol + 2.0 ** -24      # an output below 2^-14 is an fp16 subnormal
    with np.errstate(invalid="ignore"):
        ratio = float(np.nanmax(err / (UNIT[precision] * scale))) if np.isfinite(err).all() else float("inf")
    RATIOS[precision] = max(RATIOS.get(precision, 0.0), ratio)
    print("%s %s: max err / (unit * scale) = %.3f" % (what, precision, ratio))
    assert (err <= tol).all(), (what, precision, worst(err, tol))


def he(r, shape, fan_in):
    return (r.standard_normal(shape) * (2.0 / fan_in) ** 0.5).astype(np.float32)
