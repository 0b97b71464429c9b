"""The general DCNv2 forward (yb_dcn_forward_ex, dcn_v2_conv / DCN): deformable groups, any kernel size and anisotropic
geometry, judged PER ELEMENT against the float64 restatement tests/dcn_general_reference.py (checked on the CPU against
torchvision and the oracle) with the bound the existing DCN tests use: |y - ref| <= K * unit * (sum_k |w_k| * mag_k +
|bias|), mag = sum over corners of |weight * mask * x|.

Kernel by case: f32 -> dcn_simt_kernel<float> (any C); f16tc with (C/dg) % 64 == 0 -> dcn_tc_kernel<BN, false>, else
(C/dg) % 16 == 0 -> dcn_simt_kernel<__half>; f16x3 -> dcn_tc_kernel<BN, true> ((C/dg) % 64 == 0 only).
"""
import ctypes

import numpy as np
import pytest
import torch

from tests.dcn_general_reference import dcn_forward, out_size
from tests.error_bounds import UNIT, worst
from yolact_b200 import _lib
from yolact_b200.dcn_v2 import DCN, _handle, dcn_v2_conv

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1
K_BOUND = {"f16tc": 2.0, "f16x3": 4.0, "f32": 8.0}   # as tests/test_gpu_dcn_edges.py derives them
SENTINEL = -12345.0
f32 = np.float32


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def random_inputs(r, B, C, Co, H, W, kernel, stride, pad, dil, dg):
    kernel, stride, pad, dil = map(pair, (kernel, stride, pad, dil))
    Ho, Wo = out_size(H, kernel[0], stride[0], pad[0], dil[0]), out_size(W, kernel[1], stride[1], pad[1], dil[1])
    taps = kernel[0] * kernel[1]
    x = r.standard_normal((B, C, H, W)).astype(f32)
    w = (r.standard_normal((Co, C) + kernel) * (2.0 / (taps * C)) ** 0.5).astype(f32)
    bias = (r.standard_normal(Co) * 0.1).astype(f32)
    off = (r.standard_normal((B, 2 * dg * taps, Ho, Wo)) * 2.0).astype(f32)
    off[r.uniform(size=off.shape) < 0.05] *= 20
    msk = (1 / (1 + np.exp(-r.standard_normal((B, dg * taps, Ho, Wo))))).astype(f32)
    return x, off, msk, w, bias


def run(x, off, msk, w, bias, stride, pad, dil, dg, precision):
    return dcn_v2_conv(t(x), t(off), t(msk), t(w), t(bias), stride, pad, dil, dg, precision=precision).cpu().numpy()


def check(y, x, off, msk, w, bias, stride, pad, dil, dg, precision, what):
    ref, scale = dcn_forward(x, off, msk, w, bias, pair(stride), pair(pad), pair(dil), dg)
    assert y.shape == ref.shape
    err = np.abs(y - ref)
    tol = K_BOUND[precision] * UNIT[precision] * scale
    if precision == "f16tc":
        tol = tol + 2.0 ** -24
    print("%s %s: max err / (unit * scale) = %.3f" % (what, precision, (err / (UNIT[precision] * scale)).max()))
    assert (err <= tol).all(), (what, precision, worst(err, tol))


# ----------------------------------------------------------------------------------------------------------------
# a. both kernel families, every precision, groups, kernel sizes, anisotropic geometry
# ----------------------------------------------------------------------------------------------------------------
CASES = [  # precision, C, dg, Co, kernel, stride, pad, dil, H, W
    # CUDA cores, f32: any C, group boundaries inside a 16-column k-block, scalar channel tails
    ("f32", 3, 1, 5, 3, 1, 1, 1, 9, 8),
    ("f32", 24, 1, 16, 3, 1, 1, 1, 9, 8),
    ("f32", 24, 3, 16, (1, 3), (1, 2), (0, 1), 1, 9, 11),
    ("f32", 20, 4, 9, 5, (2, 1), (2, 3), (1, 2), 12, 10),
    ("f32", 6, 2, 8, 7, 1, 3, 1, 10, 9),
    ("f32", 64, 2, 64, 1, 1, 0, 1, 7, 7),
    # CUDA cores, f16tc: (C/dg) % 16 == 0 but not % 64
    ("f16tc", 64, 2, 24, 3, 1, 1, 1, 9, 8),
    ("f16tc", 48, 3, 16, (3, 1), (2, 1), (1, 0), (1, 2), 11, 9),
    ("f16tc", 32, 2, 16, 5, 1, 2, 1, 9, 9),
    # tensor cores: (C/dg) in {64, 128}, dg 2 / 4 / 8
    ("f16tc", 128, 2, 64, 3, 1, 1, 1, 10, 9),
    ("f16x3", 128, 2, 64, 3, 1, 1, 1, 10, 9),
    ("f16tc", 256, 4, 72, 3, 2, 1, 1, 13, 11),
    ("f16x3", 256, 4, 72, 3, 2, 1, 1, 13, 11),
    ("f16tc", 512, 8, 136, 3, 1, 1, 1, 8, 8),
    ("f16x3", 512, 8, 136, 3, 1, 1, 1, 8, 8),
    ("f16tc", 256, 2, 128, 3, 1, 1, 1, 9, 9),
    ("f16x3", 512, 4, 64, 3, 1, 2, 2, 9, 9),
    # tensor cores: kernel sizes and anisotropic geometry
    ("f16tc", 128, 2, 32, 1, 1, 0, 1, 9, 9),
    ("f16x3", 128, 2, 32, (1, 3), (1, 2), (0, 1), 1, 9, 11),
    ("f16tc", 128, 2, 40, 5, (2, 1), (2, 3), (1, 2), 12, 10),
    ("f16x3", 128, 2, 40, 5, (2, 1), (2, 3), (1, 2), 12, 10),
    ("f16tc", 64, 1, 24, 7, 1, 3, 1, 11, 10),
    ("f16x3", 128, 2, 24, 7, (1, 2), (3, 1), (1, 1), 11, 10),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s-C%s-dg%s-Co%s-k%s-s%s-p%s-d%s" % tuple(
    str(v).replace(" ", "") for v in c[:8]))
def test_general_forward_vs_float64(case):
    precision, C, dg, Co, kernel, stride, pad, dil, H, W = case
    args = random_inputs(np.random.RandomState(C + 7 * dg + Co), 2, C, Co, H, W, kernel, stride, pad, dil, dg)
    y = run(*args, pair(stride), pair(pad), pair(dil), dg, precision)
    check(y, *args, stride, pad, dil, dg, precision, "C=%d dg=%d" % (C, dg))


# ----------------------------------------------------------------------------------------------------------------
# b. sampling edges in a non-first group
# ----------------------------------------------------------------------------------------------------------------
def edge_targets(n):
    t = [f32(-1), f32(0), f32(n - 1), f32(n), f32(-0.5), f32(n - 0.5)]
    return np.array([v for e in t for v in (np.nextafter(e, f32(-np.inf)), e, np.nextafter(e, f32(np.inf)))], f32)


@pytest.mark.parametrize("precision,C", [("f32", 32), ("f16tc", 32), ("f16tc", 128), ("f16x3", 128)])
def test_offsets_on_and_one_ulp_around_the_edges_of_group_1(precision, C):
    """Group 1's offsets put every sample of every tap exactly on, or one ulp either side of, the places where the
    inside test, the corner tests and the floor change their answer; group 0 samples at random."""
    r = np.random.RandomState(C)
    H, W, dg = 7, 6, 2
    x, off, msk, w, bias = random_inputs(r, 2, C, 24, H, W, 3, 1, 1, 1, dg)
    Ho, Wo = off.shape[2:]
    th, tw = edge_targets(H), edge_targets(W)
    for tap in range(9):
        i, j = divmod(tap, 3)
        base_h = (np.arange(Ho)[:, None] - 1 + i).astype(f32)
        base_w = (np.arange(Wo)[None, :] - 1 + j).astype(f32)
        want_h = th[r.randint(len(th), size=(2, Ho, Wo))]
        want_w = tw[r.randint(len(tw), size=(2, Ho, Wo))]
        off[:, 18 + 2 * tap] = (want_h - base_h).astype(f32)
        off[:, 18 + 2 * tap + 1] = (want_w - base_w).astype(f32)
        reached = ((base_h + off[:, 18 + 2 * tap]).astype(f32) == want_h).mean()
        assert reached > 0.4          # most targets are reached exactly in fp32 (the restatement uses the same sums)
    msk[:, 9:] = np.where(r.uniform(size=msk[:, 9:].shape) < 0.3, f32(1.0), msk[:, 9:])
    y = run(x, off, msk, w, bias, (1, 1), (1, 1), (1, 1), dg, precision)
    check(y, x, off, msk, w, bias, 1, 1, 1, dg, precision, "edges")


# ----------------------------------------------------------------------------------------------------------------
# c. the reference script's forward checks (external/DCNv2/test.py)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,C", [("f32", 2), ("f32", 64), ("f16x3", 128)])
def test_zero_offset_identity_with_two_groups(precision, C):
    """check_zero_offset with deformable_groups = 2: zero offsets, masks sigmoid(0) = 0.5 and the identity at the
    centre tap give 2 * out == in (exactly in f32, to the hi+lo resolution in f16x3)."""
    N, H, W, dg = 2, 4, 4, 2
    x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(C)).cuda()
    off = torch.zeros(N, dg * 2 * 9, H, W, device="cuda")
    msk = torch.sigmoid(torch.zeros(N, dg * 9, H, W, device="cuda"))
    w = torch.zeros(C, C, 3, 3, device="cuda")
    w[torch.arange(C), torch.arange(C), 1, 1] = 1.0
    y = dcn_v2_conv(x, off, msk, w, torch.zeros(C, device="cuda"), 1, 1, 1, dg, precision=precision)
    d = (x - 2 * y).abs().max().item()
    assert d < (1e-10 if precision == "f32" else 1e-6 * x.abs().max().item()), d


def test_example_dconv_module_forward():
    """example_dconv: DCN(64, 64, 3, stride 1, padding 1, deformable_groups=2) on 2 x 64 x 128^2 (the CUDA-core kernel:
    32-channel groups), with the offset / mask conv seeded so that the offsets are not zero."""
    torch.manual_seed(0)
    dcn = DCN(64, 64, kernel_size=(3, 3), stride=1, padding=1, deformable_groups=2).cuda()
    with torch.no_grad():
        dcn.conv_offset_mask.weight.normal_(0, 0.05)
        dcn.conv_offset_mask.bias.normal_(0, 0.5)
    x = torch.randn(2, 64, 128, 128, device="cuda")
    with torch.no_grad():
        y = dcn(x)
        o1, o2, m = torch.chunk(dcn.conv_offset_mask(x), 3, dim=1)
        off, msk = torch.cat((o1, o2), dim=1), torch.sigmoid(m)
    assert y.shape == (2, 64, 128, 128)
    assert off.abs().mean().item() > 0.1
    n = lambda a: a.detach().cpu().numpy()
    check(n(y), n(x), n(off), n(msk), n(dcn.weight), n(dcn.bias), 1, 1, 1, 2, "f32", "example_dconv")


# ----------------------------------------------------------------------------------------------------------------
# d. yb_dcn_forward is yb_dcn_forward_ex on its own domain, bit for bit
# ----------------------------------------------------------------------------------------------------------------
def forward_old(out, x, off, msk, w, bias, s, p, d, precision):
    B, C, H, W = x.shape
    return _lib.load().yb_dcn_forward(_handle(out.device, _lib.PRECISIONS[precision]), _lib.ptr(x), _lib.ptr(w),
                                      _lib.ptr(bias), _lib.ptr(off), _lib.ptr(msk), _lib.ptr(out), B, C, H, W,
                                      w.shape[0], 3, 3, s, s, p, p, d, d, 1, _lib.current_stream(out.device))


def forward_ex(out, x, off, msk, w, bias, geom, precision, null=()):
    B, C, H, W = x.shape
    ptr = lambda name, a: ctypes.c_void_p(0) if name in null else _lib.ptr(a)
    g = None if "params" in null else ctypes.byref(_lib.YbDcnParams(*geom))
    return _lib.load().yb_dcn_forward_ex(_handle(out.device, _lib.PRECISIONS[precision]), ptr("input", x),
                                         ptr("weight", w), ptr("bias", bias), ptr("offset", off), ptr("mask", msk),
                                         ptr("output", out), B, C, H, W, w.shape[0], g, _lib.current_stream(out.device))


OLD_DOMAIN = [(C, s, p, d, Co) for C in (16, 64, 128) for (s, p, d) in ((1, 1, 1), (2, 1, 1), (1, 2, 2), (2, 0, 1))
              for Co in (5, 64)]


@pytest.mark.parametrize("precision", ["f32", "f16tc", "f16x3"])
def test_old_entry_equals_ex_bitwise(precision):
    checked = 0
    for C, s, p, d, Co in OLD_DOMAIN:
        if precision == "f16x3" and C % 64:
            continue
        r = np.random.RandomState(C + s + 3 * p + Co)
        x, off, msk, w, bias = (t(a) for a in random_inputs(r, 2, C, Co, 11, 10, 3, s, p, d, 1))
        Ho, Wo = off.shape[2:]
        y0 = torch.full((2, Co, Ho, Wo), SENTINEL, device="cuda")
        y1 = torch.full((2, Co, Ho, Wo), SENTINEL, device="cuda")
        assert forward_old(y0, x, off, msk, w, bias, s, p, d, precision) == 0, _lib.load().yb_last_error()
        assert forward_ex(y1, x, off, msk, w, bias, (3, 3, s, s, p, p, d, d, 1), precision) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(y0).all() and torch.equal(y0, y1), (C, s, p, d, Co)
        checked += 1
    assert checked >= 16


# ----------------------------------------------------------------------------------------------------------------
# e. refusals of yb_dcn_forward_ex
# ----------------------------------------------------------------------------------------------------------------
REFUSALS = [  # name, precision, C, geometry (kh, kw, sh, sw, ph, pw, dh, dw, dg), null, message
    ("kernel-0", "f32", 8, (0, 3, 1, 1, 1, 1, 1, 1, 1), (), "kernel_h and kernel_w must be >= 1"),
    ("taps-1056", "f32", 8, (33, 32, 1, 1, 1, 1, 1, 1, 1), (), "kernel_h * kernel_w <= 1024"),
    ("stride-0", "f32", 8, (3, 3, 1, 0, 1, 1, 1, 1, 1), (), "stride and dilation must be >= 1"),
    ("pad-neg", "f32", 8, (3, 3, 1, 1, -1, 1, 1, 1, 1), (), "padding >= 0"),
    ("dil-0", "f32", 8, (3, 3, 1, 1, 1, 1, 0, 1, 1), (), "stride and dilation must be >= 1"),
    ("dg-0", "f32", 8, (3, 3, 1, 1, 1, 1, 1, 1, 0), (), "deformable_group must be >= 1 and divide C"),
    ("dg-3-C8", "f32", 8, (3, 3, 1, 1, 1, 1, 1, 1, 3), (), "deformable_group must be >= 1 and divide C"),
    ("split-Cg32", "f16x3", 64, (3, 3, 1, 1, 1, 1, 1, 1, 2), (), "split-precision mode needs (C / deformable_group)"),
    ("f16-Cg8", "f16tc", 16, (3, 3, 1, 1, 1, 1, 1, 1, 2), (), "fp16 mode needs (C / deformable_group) % 16"),
    ("empty", "f32", 8, (9, 3, 1, 1, 0, 1, 1, 1, 1), (), "empty output"),
    ("null-input", "f32", 8, (3, 3, 1, 1, 1, 1, 1, 1, 1), ("input",), "null argument"),
    ("null-mask", "f32", 8, (3, 3, 1, 1, 1, 1, 1, 1, 1), ("mask",), "null argument"),
    ("null-params", "f32", 8, (3, 3, 1, 1, 1, 1, 1, 1, 1), ("params",), "null argument"),
]


@pytest.mark.parametrize("name,precision,C,geom,null,message", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_ex_refusals_return_invalid_and_leave_the_output(name, precision, C, geom, null, message):
    r = np.random.RandomState(0)
    x = t(r.standard_normal((1, C, 6, 6)).astype(f32))
    off = t(np.zeros((1, 2 * 2 * 9, 6, 6), f32))
    msk = t(np.ones((1, 2 * 9, 6, 6), f32))
    w = t(r.standard_normal((8, C, 3, 3)).astype(f32))
    out = torch.full((1, 8, 6, 6), SENTINEL, device="cuda")
    st = forward_ex(out, x, off, msk, w, t(np.zeros(8, f32)), geom, precision, null)
    assert st == YB_ERR_INVALID
    assert message in _lib.load().yb_last_error().decode()
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
    y = dcn_v2_conv(x, off[:, :18], msk[:, :9], w, t(np.zeros(8, f32)), 1, 1, 1, 1, precision=precision)
    assert torch.isfinite(y).all()
