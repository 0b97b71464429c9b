"""The network's max pool and bilinear resample kernels, through yb_resample_ex, element by element against float64
(tests/resample_reference.py), in every activation format: fp32 (precision 0), fp16 (1) and hi | lo pairs (3).

Every tensor lies between guard bands of more than one image row: the max pool's input guards hold +65504 (a stray read
wins the max), the resample's hold NaN (fmaxf would drop one); outputs start as NaN between guards of a fixed byte
pattern, so every output element must be written and nothing outside.  Three images per call, with per-image value
offsets, so that a read from the neighbouring image changes the middle image's result too.

  max pool:  bit for bit against the encoding of the float64 max (the max, the re-encode and the inputs are exact), at
             the stem output sizes of the configs and 1..7-pixel maps, with the window maxima on border taps, all-negative
             corner windows and, in split mode, windows whose hi planes tie and whose lo planes decide;
  bilinear:  within K * unit * (sum |lambda * p| + |add|) at the FPN's top-down resizes (with the lateral add), the
             protonet's x2 + ReLU on mixed-sign input, and edge shapes; in split mode the bound is tight enough that
             dropping the output's lo plane (a 2^-11 relative error) fails it.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests import resample_reference as R
from tests.error_bounds import U16, U22, U24, worst
from yolact_b200 import _lib

pytestmark = pytest.mark.gpu

PRECISION = {"f32": 0, "f16": 1, "f16x3": 3}          # yb_resample_ex's precision argument
DTYPE = {"f32": np.float32, "f16": np.float16, "f16x3": np.float16}
VEC = {"f32": 4, "f16": 8, "f16x3": 8}                  # channels per 16-byte vector
UNIT = {"f32": U24, "f16": U16, "f16x3": U22}
# f32:   the products and the three sums of the blend and the add (1 unit each of the partial magnitude)
# f16:   the fp16 rounding of the output (1 unit); the fp32 blend adds a 2^-13 fraction of a unit
# f16x3: the hi / lo encoding of the output (1 unit) + the fp32 blend (4 * 2^-24 = 1 unit)
K_BOUND = {"f32": 4.0, "f16": 1.25, "f16x3": 3.0}
GUARD_BYTE = 0x5A
B = 3
PRECS = ["f32", "f16", "f16x3"]

RATIOS = {}   # precision -> largest err / (unit * scale) of the resample


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    for prec in sorted(RATIOS):
        print("bilinear: largest err / (unit * scale), %s: %.3f" % (prec, RATIOS[prec]))


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


def guarded_input(raw, guard, guard_px):
    """raw [B, H, W, PS] (kernel dtype) on the device between two bands of `guard` pixels equal to guard_px."""
    PS = raw.shape[-1]
    n = raw.size // PS
    host = np.empty((n + 2 * guard, PS), raw.dtype)
    host[:guard] = guard_px
    host[guard + n:] = guard_px
    host[guard:guard + n] = raw.reshape(n, PS)
    return torch.from_numpy(host).cuda()[guard:guard + n]


def guarded_output(shape, dtype, guard):
    """A device buffer of `shape` full of NaN (0xff bytes) between two bands of GUARD_BYTE; returns (buffer, view)."""
    PS = shape[-1]
    n = int(np.prod(shape[:-1]))
    buf = torch.empty((n + 2 * guard, PS), dtype=torch.float32 if dtype == np.float32 else torch.float16, device="cuda")
    buf.view(torch.uint8).fill_(GUARD_BYTE)
    buf[guard:guard + n].view(torch.uint8).fill_(0xFF)
    return buf, buf[guard:guard + n]


def call(hd, op, prec, x, add, y, H, W, C, Ho, Wo, relu):
    lib, h = hd
    _lib.check(lib.yb_resample_ex(h, op, PRECISION[prec], _lib.ptr(x), _lib.ptr(add), _lib.ptr(y), B, H, W, C, Ho, Wo,
                                  relu, _lib.current_stream()), "yb_resample_ex")
    torch.cuda.synchronize()


def run(hd, op, prec, x_raw, in_guard_px, Ho, Wo, add_raw=None, relu=0):
    """One yb_resample_ex call on guarded buffers; returns the raw output [B, Ho, Wo, PS] as numpy."""
    _, H, W, PS = x_raw.shape
    C = PS // 2 if prec == "f16x3" else PS
    guard = max(W, Wo) + 2          # one image row plus one pixel, and more
    x = guarded_input(x_raw, guard, in_guard_px)
    add = None if add_raw is None else guarded_input(add_raw, guard, in_guard_px)
    buf, y = guarded_output((B, Ho, Wo, PS), DTYPE[prec], guard)
    call(hd, op, prec, x, add, y, H, W, C, Ho, Wo, relu)
    bands = torch.cat([buf[:guard], buf[-guard:]]).view(torch.uint8)
    assert (bands == GUARD_BYTE).all(), "%d guard bytes of the output changed" % (bands != GUARD_BYTE).sum().item()
    return y.view(B, Ho, Wo, PS).cpu().numpy()


def encoded_pixel(v, prec, C):
    return R.encode_nhwc(np.full((C,), v, np.float32), prec)


# ----------------------------------------------------------------------------------------------------------------
# max pool 3x3 / 2 / pad 1
# ----------------------------------------------------------------------------------------------------------------
def maxpool_input(H, W, C, prec, seed):
    """Mixed signs; per-image offsets 0, -16, +16 (the middle image lies below both neighbours, so a read from either
    wins); a third of the border pixels raised by 30 (the window maximum on a border tap); the corner windows all
    negative.  Split mode: values within 0.45 ulp of a half-integer hi, so that the hi planes of a window tie often and
    the lo' planes decide among them."""
    r = np.random.RandomState(seed)
    v = r.standard_normal((B, H, W, C)) * 4 + np.array([0.0, -16.0, 16.0])[:, None, None, None]
    border = np.zeros((H, W), bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    v = np.where(border[None, :, :, None] & (r.uniform(size=v.shape) < 1 / 3), v + 30, v)
    for rows in (slice(0, 2), slice(max(H - 3, 0), H)):
        for cols in (slice(0, 2), slice(max(W - 3, 0), W)):
            v[:, rows, cols] = -1 - np.abs(v[:, rows, cols])
    if prec != "f16x3":
        return R.encode_nhwc(v, prec)
    hi = (np.floor(v) + 0.5).astype(np.float16)
    ulp = np.spacing(np.abs(hi)).astype(np.float32)
    return R.encode_nhwc(hi.astype(np.float32) + r.uniform(-0.45, 0.45, v.shape).astype(np.float32) * ulp, prec)


MAXPOOL_STEM = [(275, 275), (350, 350), (80, 80), (128, 160)]   # the stem outputs of the 550, 700, 160, 256x320 inputs
MAXPOOL_SMALL = [(1, 1), (1, 2), (2, 1), (3, 3), (5, 7)]


def check_maxpool(hd, H, W, C, prec):
    x_raw = maxpool_input(H, W, C, prec, H * 1000 + W + C)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    got = run(hd, _lib.YB_RESAMPLE_MAXPOOL, prec, x_raw, encoded_pixel(65504.0, prec, C), Ho, Wo)
    want = R.encode_nhwc(R.maxpool3x3s2_f64(R.decode_nhwc(x_raw, prec)), prec)
    bits = np.uint32 if prec == "f32" else np.uint16
    bad = got.view(bits) != want.view(bits)
    if bad.any():
        at = tuple(np.argwhere(bad)[0])
        pytest.fail("maxpool %dx%dx%d %s: %d elements differ; first at %s: got %r want %r"
                    % (H, W, C, prec, bad.sum(), at, got[at], want[at]))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("H,W", MAXPOOL_STEM, ids=str)
def test_maxpool_stem_outputs(hd, H, W, prec):
    check_maxpool(hd, H, W, 64, prec)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("C", ["vec", 64])
@pytest.mark.parametrize("H,W", MAXPOOL_SMALL, ids=str)
def test_maxpool_small_maps(hd, H, W, C, prec):
    check_maxpool(hd, H, W, VEC[prec] if C == "vec" else C, prec)


def test_maxpool_split_ties_are_decided_by_lo():
    """The split case's input really has windows whose largest hi is held by several taps, so that the lo planes decide
    the maximum, of both signs (checked on the reference: a pool comparing hi alone cannot pass by luck)."""
    x_raw = maxpool_input(80, 80, 64, "f16x3", 80 * 1000 + 80 + 64)
    hi = x_raw[..., :64].astype(np.float64)
    hi_max = R.maxpool3x3s2_f64(hi)
    Ho = hi_max.shape[1]
    hp = np.full((B, 2 * Ho + 1, 2 * Ho + 1, 64), -np.inf)
    hp[:, 1:81, 1:81] = hi
    ties = sum((hp[:, r:r + 2 * Ho:2, s:s + 2 * Ho:2] == hi_max).astype(int) for r in range(3) for s in range(3))
    tied = ties >= 2
    assert tied.mean() > 0.05
    assert (tied & (hi_max > 0)).sum() > 1000 and (tied & (hi_max < 0)).sum() > 1000


# ----------------------------------------------------------------------------------------------------------------
# bilinear resample, align_corners=False
# ----------------------------------------------------------------------------------------------------------------
def bilinear_case(H, W, Ho, Wo, C, prec, with_add, seed):
    """Inputs and add N(0, 2) plus per-image offsets -1.5, 0, +1.5 (mixed signs in every image)."""
    r = np.random.RandomState(seed)
    off = np.array([-1.5, 0.0, 1.5])[:, None, None, None]
    x_raw = R.encode_nhwc(r.standard_normal((B, H, W, C)) * 2 + off, prec)
    add_raw = R.encode_nhwc(r.standard_normal((B, Ho, Wo, C)) * 2 - off, prec) if with_add else None
    return x_raw, add_raw


def check_bilinear(hd, H, W, Ho, Wo, C, prec, with_add, relu):
    x_raw, add_raw = bilinear_case(H, W, Ho, Wo, C, prec, with_add, H * 7919 + Wo * 31 + C)
    got_raw = run(hd, _lib.YB_RESAMPLE_BILINEAR, prec, x_raw, encoded_pixel(np.nan, prec, C), Ho, Wo, add_raw, relu)
    got = R.decode_nhwc(got_raw, prec)
    want, scale = R.bilinear_f64(R.decode_nhwc(x_raw, prec), Ho, Wo,
                                 None if add_raw is None else R.decode_nhwc(add_raw, prec), bool(relu))
    if relu:   # the case exercises the ReLU: many outputs are clamped
        pre, _ = R.bilinear_f64(R.decode_nhwc(x_raw, prec), Ho, Wo,
                                None if add_raw is None else R.decode_nhwc(add_raw, prec))
        assert (pre < -100 * UNIT[prec] * scale).mean() > 0.1
    err = np.abs(got - want)
    tol = K_BOUND[prec] * UNIT[prec] * scale
    if prec == "f16":
        tol = tol + 2.0 ** -25      # an output below 2^-14 is an fp16 subnormal
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = float(np.nanmax(np.where(scale > 0, err / (UNIT[prec] * scale), 0))) if np.isfinite(err).all() else np.inf
    RATIOS[prec] = max(RATIOS.get(prec, 0.0), ratio)
    what = "bilinear %dx%d -> %dx%d C=%d %s%s%s" % (H, W, Ho, Wo, C, prec, " +add" if with_add else "",
                                                  " relu" if relu else "")
    print("%s: max err / (unit * scale) = %.3f" % (what, ratio))
    assert (err <= tol).all(), (what, worst(err, tol))
    if prec == "f16x3":   # the bound resolves the lo plane: the output's hi plane alone misses it
        hi_only = got_raw[..., :C].astype(np.float64)
        nz = want != 0
        assert (np.abs(hi_only - want)[nz] > tol[nz]).mean() > 0.5, what


FPN_RESIZES = [((18, 18), (35, 35)), ((35, 35), (69, 69)),     # 550
               ((22, 22), (44, 44)), ((44, 44), (88, 88)),     # 700
               ((5, 5), (10, 10)), ((10, 10), (20, 20)),       # 160
               ((8, 10), (16, 20)), ((16, 20), (32, 40))]      # 256x320 frames
PROTO_RESIZES = [((69, 69), (138, 138)), ((88, 88), (176, 176)), ((35, 35), (70, 70))]
EDGE_RESIZES = [((1, 1), (2, 2)), ((1, 7), (3, 13)), ((9, 5), (17, 11)), ((12, 12), (12, 12))]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("src,dst", FPN_RESIZES, ids=str)
def test_bilinear_fpn_top_down_with_lateral(hd, src, dst, prec):
    check_bilinear(hd, *src, *dst, 256, prec, with_add=True, relu=0)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("src,dst", PROTO_RESIZES, ids=str)
def test_bilinear_protonet_x2_relu(hd, src, dst, prec):
    check_bilinear(hd, *src, *dst, 64, prec, with_add=False, relu=1)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("src,dst", EDGE_RESIZES, ids=str)
def test_bilinear_edge_shapes(hd, src, dst, relu, prec):
    check_bilinear(hd, *src, *dst, VEC[prec] * 2, prec, with_add=True, relu=relu)


# ----------------------------------------------------------------------------------------------------------------
# refusals
# ----------------------------------------------------------------------------------------------------------------
REFUSALS = {   # name -> (op, precision, C, H, W, Ho, Wo, with_add, relu)
    "precision-2": (1, 2, 8, 4, 4, 8, 8, False, 0),
    "precision-4": (1, 4, 8, 4, 4, 8, 8, False, 0),
    "precision-negative": (0, -1, 8, 4, 4, 2, 2, False, 0),
    "f32-C-6": (1, 0, 6, 4, 4, 8, 8, False, 0),
    "f16-C-4": (1, 1, 4, 4, 4, 8, 8, False, 0),
    "split-C-12": (0, 3, 12, 4, 4, 2, 2, False, 0),
    "maxpool-Ho": (0, 0, 8, 5, 5, 2, 3, False, 0),
    "maxpool-Wo": (0, 1, 8, 5, 5, 3, 4, False, 0),
    "maxpool-add": (0, 0, 8, 4, 4, 2, 2, True, 0),
    "maxpool-relu": (0, 3, 8, 4, 4, 2, 2, False, 1),
    "unknown-op": (2, 0, 8, 4, 4, 8, 8, False, 0),
}


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals_launch_nothing(hd, name):
    lib, h = hd
    op, prec, C, H, W, Ho, Wo, with_add, relu = REFUSALS[name]
    x = torch.zeros(B * H * W * 2 * C, device="cuda")
    add = torch.zeros(B * Ho * Wo * 2 * C, device="cuda") if with_add else None
    y = torch.zeros(B * Ho * Wo * 2 * C, device="cuda")
    before = lib.yb_launch_count(h)
    with pytest.raises(_lib.YbError):
        _lib.check(lib.yb_resample_ex(h, op, prec, _lib.ptr(x), _lib.ptr(add), _lib.ptr(y), B, H, W, C, Ho, Wo, relu,
                                      _lib.current_stream()), "yb_resample_ex")
    assert lib.yb_launch_count(h) == before
    assert (y == 0).all()
