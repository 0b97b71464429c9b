"""The fused DCNv2 kernels sample by sample at the sampling edges, at the layer shapes YOLACT++ runs, and at the tile
and channel edges -- every case against a float64 blend of the reference's corners (oracle.dcn_v2_columns,
acc=np.float64; checked on the CPU by tests/test_dcn_reference_host.py) and judged PER ELEMENT against the magnitude
the arithmetic's rounding is proportional to, so one dropped or misplaced corner cannot hide under a range bound.

Kernel by case: C % 64 == 0 in f16tc / f16x3 -> dcn_tc_kernel<BN, SPLIT> (tensor cores); C = 32 in f16tc ->
dcn_simt_kernel<__half>; f32 -> dcn_simt_kernel<float>.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

from oracle import yolact_oracle as O
from tests.dcn_probe import GEOMETRIES, build_probe_case, out_hw, selected_columns
from tests.error_bounds import UNIT, worst
from yolact_b200 import _lib
from yolact_b200.dcn_v2 import _handle, dcn_v2_conv

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1       # include/yolact_b200.h
# Whole-output bound, per element: |y - ref| <= K * unit * scale, scale = sum_k |w_k| * mag_k + |bias|, where
# mag = sum over corners |weight * mask * x| is what a rounding error of one sample is proportional to.
#  f16tc  1 for the fp16 rounding of the output (coherent: |y| <= scale) + 1 for the roundings of the operands -- x,
#         the folded corner weight, the four half2 blend steps, the fp16 weight: up to 7 units per TERM, but of
#         independent sign over the 9*C >= 576 terms, so they add like sqrt(9*C), a small fraction of the sum.
#         Measured on an H100: at most 0.61.
#  f16x3  the same count in units of 2^-22 (one hi+lo encoding: the lo half is an fp16 rounding of a residual of at
#         most 2^-11 |v|; x, sample, weight and output are each encoded once), + 2 for
#         the fp32 blend (6 roundings of 2^-24) and the fp32 accumulation over up to 4608 terms (2^-24 = 1/4 unit
#         each, random-signed).  Measured: at most 2.4, at C = 512.
#  f32    the blend's 6 fp32 roundings per term and the sequential fp32 accumulation, random-signed over the terms:
#         a sequential fp32 sum of the same products on the CPU reaches 5.0 over the 1.2 M outputs of the largest
#         case, the kernel 6.0.
K_BOUND = {"f16tc": 2.0, "f16x3": 4.0, "f32": 8.0}


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(x, off, msk, w, bias, stride, pad, dil, precision):
    return dcn_v2_conv(t(x), t(off), t(msk), t(w), t(bias), stride, pad, dil, 1, precision=precision).cpu().numpy()


def random_inputs(r, B, C, Co, H, W, stride, pad=1, dil=1):
    """He-scaled weights, offsets N(0, 2) with 5 % of them scaled x20 (whole taps fall outside), sigmoid masks."""
    Ho, Wo = out_hw(H, W, stride, pad, dil)
    x = r.standard_normal((B, C, H, W)).astype(np.float32)
    w = (r.standard_normal((Co, C, 3, 3)) * (2.0 / (9 * C)) ** 0.5).astype(np.float32)
    bias = (r.standard_normal(Co) * 0.1).astype(np.float32)
    off = (r.standard_normal((B, 18, Ho, Wo)) * 2.0).astype(np.float32)
    off[r.uniform(size=off.shape) < 0.05] *= 20
    msk = (1 / (1 + np.exp(-r.standard_normal((B, 9, Ho, Wo))))).astype(np.float32)
    return x, off, msk, w, bias


def reference(x, off, msk, w, bias, stride, pad, dil):
    """float64 output and the per-element scale sum_k |w_k| * mag_k + |bias| of its rounding error."""
    cols, mag = O.dcn_v2_columns(x, off, msk, stride, pad, dil, acc=np.float64, with_abs=True)
    ref = O.dcn_v2_contract(cols, w, bias, acc=np.float64)
    scale = O.dcn_v2_contract(mag, np.abs(w), np.abs(bias), acc=np.float64)
    return ref, scale


def check_output(y, ref, scale, precision, what):
    assert y.shape == ref.shape
    err = np.abs(y - ref)
    tol = K_BOUND[precision] * UNIT[precision] * scale
    if precision == "f16tc":
        tol = tol + 2.0 ** -24      # an output below 2^-14 is an fp16 subnormal
    print("%s %s: max err / (unit * scale) = %.3f" % (what, precision, (err / (UNIT[precision] * scale)).max()))
    assert (err <= tol).all(), (what, precision, worst(err, tol))
    if precision == "f16x3":
        assert err.max() < 2e-5 * max(1.0, np.abs(ref).max())


# ----------------------------------------------------------------------------------------------------------------
# a. sampling probe: selection-matrix weights, the output is the column
# ----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def probe(geometry, C):
    s, pad, dil, H, W = geometry
    case = build_probe_case(H, W, s, pad, dil, C, seed=100 * H + 10 * s + pad)
    cols, mag = O.dcn_v2_columns(case["x"], case["offset"], case["mask"], s, pad, dil, acc=np.float64, with_abs=True)
    return case, selected_columns(cols, case), selected_columns(mag, case)


@pytest.mark.parametrize("C,precision", [(64, "f16tc"), (64, "f16x3"), (64, "f32"), (32, "f16tc"), (32, "f32")])
@pytest.mark.parametrize("geometry", GEOMETRIES, ids=lambda g: "s%d-p%d-d%d-%dx%d" % g)
def test_sampling_probe_column_by_column(geometry, C, precision):
    case, want, mag = probe(geometry, C)
    s, pad, dil = geometry[:3]
    y = run(case["x"], case["offset"], case["mask"], case["weight"], case["bias"], s, pad, dil, precision)
    xmax = float(np.abs(case["x"]).max())
    # per sample: f32 -- 4 products, 3 sums and the mask product in fp32, against the float64 blend of the same
    # corners; f16x3 -- hi+lo encodings of x, of the sample and of the output (at most 2^-22 each) + the fp32 blend
    # with the mask folded into the weights (6 roundings of 2^-24): 4.5 * 2^-22 < 2^-19; f16tc -- fp16 x and fp16 folded weight (2^-11 each) and
    # the half2 blend (2^-9 in all); a folded weight or a sample below 2^-14 is an fp16 subnormal with an absolute
    # step of 2^-24 (mask 1e-6), which the last two terms cover.
    tol = {"f32": 2.0 ** -21 * mag,
           "f16x3": 2.0 ** -19 * mag + 2.0 ** -30,
           "f16tc": 2.0 ** -9 * mag + 2.0 ** -23 * xmax + 2.0 ** -22}[precision]
    err = np.abs(y - want)
    ok = err <= tol                                  # NaN compares false
    if not ok.all():
        b, o, ho, wo = np.unravel_index(np.argmax(np.where(ok, 0, np.where(np.isfinite(err), err, np.inf))), err.shape)
        tap, c = case["sel"][o]
        pytest.fail("%d samples wrong; worst: image %d pixel (%d, %d) tap %d channel %d: got %r want %r tol %.3g, offset "
                    "(%r, %r) from base (%d, %d), mask %r"
                    % ((~ok).sum(), b, ho, wo, tap, c, y[b, o, ho, wo], want[b, o, ho, wo], tol[b, o, ho, wo],
                       case["offset"][b, 2 * tap, ho, wo], case["offset"][b, 2 * tap + 1, ho, wo],
                       case["base_h"][ho, tap], case["base_w"][wo, tap], case["mask"][b, tap, ho, wo]))
    # the whole-tensor bounds the modes promise
    assert err.max() <= {"f32": 1e-6, "f16x3": 4e-6, "f16tc": 2.0 ** -9 * 1.01}[precision] * xmax
    # outside, far outside and non-finite positions are exact zeros
    assert (y[mag == 0] == 0).all()


# ----------------------------------------------------------------------------------------------------------------
# b. a non-finite pixel reaches only the samples that read it
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("poison", [float("nan"), 7e4], ids=["nan", "7e4"])
@pytest.mark.parametrize("C,precision", [(64, "f16tc"), (64, "f16x3"), (32, "f16tc"), (64, "f32")])
def test_nonfinite_pixel_does_not_leak(C, precision, poison):
    """x[b, :, 0, 0] = NaN (or 7e4, beyond the fp16 range): every output pixel none of whose nine samples has pixel
    (0, 0) among its in-range corners -- samples wholly outside the image included -- equals, bit for bit, the result
    of a finite input.  The tensor-core kernel points every corner the reference skips, and every sample outside the
    image, at pixel 0 of the image with weight 0, so this holds only because that pixel is finite when the kernel
    reads it: the fp16 and hi+lo conversions of the input saturate (7e4 -> 65504, NaN -> -65504), which the last
    assertion pins.  In f32 the NaN stays a NaN and reaches exactly the pixels that read it, as in the reference."""
    H, W, B = 21, 19, 2
    x, off, msk, w, bias = random_inputs(np.random.RandomState(11), B, C, 24, H, W, 1)
    h_im, w_im, valid = O.dcn_v2_positions(off, H, W, 1, 1, 1)
    with np.errstate(invalid="ignore"):
        reads00 = valid & (np.floor(h_im) <= 0) & (np.floor(w_im) <= 0)     # [B, 9, Ho, Wo]
    clean = ~reads00.any(axis=1)                                            # [B, Ho, Wo]
    border = valid & ((h_im < 0) | (w_im < 0) | (h_im > H - 1) | (w_im > W - 1))
    assert clean.mean() > 0.8 and (~valid & clean[:, None]).sum() > 100 and (border & clean[:, None]).sum() > 100
    y0 = run(x, off, msk, w, bias, 1, 1, 1, precision)
    xp = x.copy()
    xp[:, :, 0, 0] = poison
    y1 = run(xp, off, msk, w, bias, 1, 1, 1, precision)
    sel = np.broadcast_to(clean[:, None], y0.shape)
    assert np.isfinite(y0).all()
    leaked = sel & (y0.view(np.uint32) != y1.view(np.uint32))
    assert not leaked.any(), "%d outputs of %d pixels that never read pixel (0, 0) changed; %d of them are not finite" % (
        leaked.sum(), leaked.any(axis=1).sum(), (leaked & ~np.isfinite(y1)).sum())
    assert (y0[~sel] != y1[~sel]).any()      # the pixels that do read it see the change
    if precision == "f32" and np.isnan(poison):
        assert np.isnan(y1[~sel]).any()
    else:
        assert np.isfinite(y1).all()


# ----------------------------------------------------------------------------------------------------------------
# c. the shapes YOLACT++ runs (input 550: 69^2 / 35^2 / 18^2 after stages 2..4; input 700: 44^2 after stage 3)
# ----------------------------------------------------------------------------------------------------------------
LAYER_SHAPES = [   # C = Co, H = W, stride, B
    (128, 138, 2, 2),   # stage-2 first block, 69^2 out
    (128, 69, 1, 3),    # M = 14283, not a multiple of 128
    (256, 35, 1, 3),    # 2 N tiles, 36 k-blocks
    (512, 18, 1, 2),    # 4 N tiles, 72 k-blocks
    (512, 35, 2, 2),    # stage-4 first block
    (256, 44, 1, 2),    # input 700
]


@functools.lru_cache(maxsize=1)
def layer_case(shape):
    C, H, stride, B = shape
    args = random_inputs(np.random.RandomState(C + H), B, C, C, H, H, stride)
    return args, reference(*args, stride, 1, 1)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3", "f32"])
@pytest.mark.parametrize("shape", LAYER_SHAPES, ids=lambda s: "C%d-%dx%d-s%d-B%d" % (s[0], s[1], s[1], s[2], s[3]))
def test_layer_shapes_vs_float64(shape, precision):
    args, (ref, scale) = layer_case(shape)
    check_output(run(*args, shape[2], 1, 1, precision), ref, scale, precision, "C=%d %d^2 s%d" % shape[:3])


# ----------------------------------------------------------------------------------------------------------------
# d. tile and channel edges
# ----------------------------------------------------------------------------------------------------------------
def forward_into(out, x, off, msk, w, bias, stride, pad, dil, precision, kernel=3, groups=1, null=()):
    """yb_dcn_forward into a caller-owned buffer (dcn_v2_conv allocates its own); returns the status.  stride, pad
    and dil are (h, w) pairs; the arguments named in `null` are passed as null pointers."""
    B, C, H, W = x.shape
    p = lambda name, a: ctypes.c_void_p(0) if name in null else _lib.ptr(a)
    return _lib.load().yb_dcn_forward(_handle(out.device, _lib.PRECISIONS[precision]), p("input", x), p("weight", w),
                                      p("bias", bias), p("offset", off), p("mask", msk), p("output", out), B, C, H, W,
                                      w.shape[0], kernel, kernel, stride[0], stride[1], pad[0], pad[1], dil[0], dil[1],
                                      groups, _lib.current_stream(out.device))


SENTINEL = -12345.0


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (1, 127, 1), (2, 8, 8), (1, 43, 3), (5, 10, 5)],
                         ids=["M1", "M127-W1", "M128", "M129", "M250-3-images-per-tile"])
def test_m_tile_edges(B, H, W, precision):
    args = random_inputs(np.random.RandomState(B * H + W), B, 64, 24, H, W, 1)
    check_output(run(*args, 1, 1, 1, precision), *reference(*args, 1, 1, 1), precision, "M=%d" % (B * H * W))


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("Co", [1, 8, 64, 72, 129, 200, 256])
def test_output_channel_edges_and_guard_band(Co, precision):
    """Co = 129 runs padded to 136 and Co = 200 as it is: both end in a partial second N tile (n0 = 128).  The padded
    channels and the rows past M (M = 144: the second M tile has 16 rows) must not reach the caller's tensor: the
    output is followed by a guard band that has to stay untouched."""
    B, H, W = 2, 9, 8
    args = random_inputs(np.random.RandomState(Co), B, 64, Co, H, W, 1)
    n = B * Co * H * W
    buf = torch.full((n + 4096,), SENTINEL, device="cuda", dtype=torch.float32)
    st = forward_into(buf, *[t(a) for a in args], (1, 1), (1, 1), (1, 1), precision)
    assert st == 0, _lib.load().yb_last_error()
    torch.cuda.synchronize()
    assert (buf[n:] == SENTINEL).all()
    y = buf[:n].view(B, Co, H, W).cpu().numpy()
    check_output(y, *reference(*args, 1, 1, 1), precision, "Co=%d" % Co)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
def test_same_handle_alternating_shapes_is_bitwise_repeatable(precision):
    r = np.random.RandomState(5)
    first = random_inputs(r, 2, 64, 136, 12, 11, 1)
    second = random_inputs(r, 1, 128, 40, 17, 9, 2)
    y1 = run(*first, 1, 1, 1, precision)
    y2 = run(*second, 2, 1, 1, precision)
    y3 = run(*first, 1, 1, 1, precision)
    assert np.isfinite(y2).all()
    assert np.array_equal(y1.view(np.uint32), y3.view(np.uint32))


# ----------------------------------------------------------------------------------------------------------------
# e. refusals
# ----------------------------------------------------------------------------------------------------------------
def _refusal_inputs(C=64, k=3):
    r = np.random.RandomState(0)
    x = t(r.standard_normal((1, C, 6, 6)).astype(np.float32))
    off = t(np.zeros((1, 2 * k * k, 6, 6), np.float32))
    msk = t(np.ones((1, k * k, 6, 6), np.float32))
    w = t(r.standard_normal((8, C, k, k)).astype(np.float32))
    return x, off, msk, w, t(np.zeros(8, np.float32))


@pytest.mark.parametrize("what,message", [
    ("stride", "anisotropic"), ("pad", "anisotropic"), ("dil", "anisotropic"),
    ("groups", "deformable_group must be 1"), ("k1", "only 3x3 kernels"), ("k5", "only 3x3 kernels"),
    ("C24", "C must be a multiple of 16"), ("split-C32", "split-precision mode needs C % 64 == 0"),
    ("null-input", "null argument"), ("null-offset", "null argument"), ("null-output", "null argument"),
])
def test_refusals_return_invalid_and_leave_the_output(what, message):
    kw = dict(stride=(1, 1), pad=(1, 1), dil=(1, 1), precision="f16tc")
    C, k = {"C24": 24, "split-C32": 32}.get(what, 64), {"k1": 1, "k5": 5}.get(what, 3)
    if what in ("stride", "pad", "dil"):
        kw[what] = (1, 2)
    if what == "groups":
        kw["groups"] = 2
    if what == "split-C32":
        kw["precision"] = "f16x3"
    if what.startswith("null-"):
        kw["null"] = (what[5:],)
    x, off, msk, w, bias = _refusal_inputs(C, k)
    out = torch.full((1, 8, 6, 6), SENTINEL, device="cuda")
    st = forward_into(out, x, off, msk, w, bias, kernel=k, **kw)
    assert st == YB_ERR_INVALID
    assert message in _lib.load().yb_last_error().decode()
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
    # the handle is still good
    x, off, msk, w, bias = _refusal_inputs()
    y = dcn_v2_conv(x, off, msk, w, bias, 1, 1, 1, 1, precision="f16tc")
    assert torch.isfinite(y).all()
