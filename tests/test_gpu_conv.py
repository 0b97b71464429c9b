"""Convolution kernels through the C ABI (yb_conv2d): SIMT fp32 vs torch fp32; tensor-core (wgmma) fp16 and the SIMT
fp16 kernel element by element against float64 on the same fp16-rounded operands, and against each other; the split
mode against float64 on the unrounded operands (the per-element bound of tests/conv_reference.py)."""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.conv_reference import K_BOUND, UNIT, act_f64, check, conv_f64, f16, report_ratios  # noqa: F401
from tests.error_bounds import worst
from yolact_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    lib = _lib.load()
    yc = _lib.YbConfig()
    yc.backbone = _lib.YB_BACKBONE_NONE
    yc.num_classes, yc.mask_dim, yc.precision = 81, 32, _lib.YB_PREC_F32
    yc.nms_top_k, yc.nms_conf_thresh, yc.nms_thresh, yc.max_num_detections = 200, 0.05, 0.5, 100
    h = ctypes.c_void_p()
    _lib.check(lib.yb_create(ctypes.byref(yc), 0, ctypes.byref(h)), "yb_create")
    yield lib, h
    lib.yb_destroy(h)


def run_conv(ops, x, w, bias, res, stride, pad, act, precision, iters=1):
    lib, h = ops
    B, Ci, H, W = x.shape
    Co, _, kh, kw = w.shape
    Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    xd = x.cuda().contiguous()
    y = torch.empty(B, Co, Ho, Wo, device="cuda")
    wc = w.contiguous()
    bc = bias.contiguous() if bias is not None else None
    rd = res.cuda().contiguous() if res is not None else None
    ms = ctypes.c_float(0)
    _lib.check(lib.yb_conv2d(h, _lib.ptr(xd), ctypes.c_void_p(wc.data_ptr()),
                             ctypes.c_void_p(bc.data_ptr()) if bc is not None else None, _lib.ptr(rd), _lib.ptr(y),
                             B, Ci, H, W, Co, kh, kw, stride, pad, act, precision, iters, ctypes.byref(ms),
                             _lib.current_stream()), "yb_conv2d")
    torch.cuda.synchronize()
    return y.cpu(), ms.value


def ref_conv(x, w, bias, res, stride, pad, act):
    y = F.conv2d(x, w, bias, stride=stride, padding=pad)
    if res is not None:
        y = y + res
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = torch.tanh(y)
    elif act == 3:
        y = F.leaky_relu(y, 0.1)
    return y


def make(B, Ci, H, W, Co, k, stride, pad, with_bias=True, with_res=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5
    bias = torch.randn(Co, generator=g) * 0.1 if with_bias else None
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = torch.randn(B, Co, Ho, Wo, generator=g) if with_res else None
    return x, w, bias, res


SIMT_CASES = [
    # B, Ci, H, W, Co, k, s, p, act, res
    (2, 3, 37, 41, 64, 7, 2, 3, 1, False),      # stem-like
    (1, 64, 19, 23, 256, 1, 1, 0, 0, True),
    (2, 48, 17, 15, 40, 3, 1, 1, 1, False),
    (1, 32, 20, 20, 24, 3, 2, 1, 3, False),
    (3, 1, 30, 30, 8, 3, 2, 0, 1, False),       # maskiou-like (no padding)
    (1, 128, 9, 9, 81, 1, 1, 0, 2, False),
]


@pytest.mark.parametrize("case", SIMT_CASES)
def test_simt_f32_matches_torch(ops, case):
    B, Ci, H, W, Co, k, s, p, act, wr = case
    x, w, bias, res = make(B, Ci, H, W, Co, k, s, p, True, wr)
    y, _ = run_conv(ops, x, w, bias, res, s, p, act, 0)
    ref = ref_conv(x, w, bias, res, s, p, act)
    assert (y - ref).abs().max() < 2e-4 * max(1.0, ref.abs().max().item())


TC_CASES = [
    # B, Ci, H, W, Co, k, s, p, act, res          (every shape family of the network, incl. odd sizes)
    (2, 64, 35, 35, 256, 1, 1, 0, 1, True),      # bottleneck conv3 + residual + relu (flattened 1x1)
    (2, 256, 35, 35, 256, 3, 1, 1, 1, False),    # 3x3 s1 (stage 3 work-horse)
    (1, 128, 69, 69, 128, 3, 2, 1, 1, False),    # 3x3 s2, odd input (phase views)
    (1, 128, 138, 138, 128, 3, 2, 1, 1, False),  # 3x3 s2, even input
    (2, 512, 69, 69, 1024, 1, 2, 0, 0, False),   # 1x1 s2 downsample (strided view)
    (2, 256, 18, 18, 243, 3, 1, 1, 0, False),    # conf head, Cout = 243
    (2, 256, 9, 9, 12, 3, 1, 1, 0, False),       # bbox head, Cout = 12
    (2, 256, 5, 5, 96, 3, 1, 1, 2, False),       # mask head, tanh
    (1, 256, 37, 23, 27, 3, 1, 1, 0, False),     # DCN offset conv, non-square
    (1, 256, 138, 138, 32, 1, 1, 0, 1, False),   # proto 1x1 -> 32
    (1, 2048, 18, 18, 256, 1, 1, 0, 0, False),   # FPN lateral, K = 2048
    (1, 256, 9, 9, 256, 3, 2, 1, 0, False),      # FPN downsample 9 -> 5
    (1, 64, 138, 138, 64, 3, 1, 1, 1, False),    # stage 1 3x3
    (1, 1152, 20, 20, 128, 1, 1, 0, 1, False),   # DCN contraction as 1x1 over 9*C columns
    (1, 64, 20, 20, 32, 1, 1, 0, 3, False),      # Darknet block conv1: fp16 output narrower than the 64-channel store box
    (2, 256, 35, 35, 1024, 1, 1, 0, 1, True),    # stage-3 conv3: 16 residual/output chunks per tile row
    (1, 256, 69, 69, 72, 3, 1, 1, 1, False),     # Cout = 72: last chunk is 8 channels wide
    (1, 128, 69, 69, 512, 1, 1, 0, 1, True),     # stage-2 conv3: 1x1 + residual, 4-8 N tiles
    (1, 512, 18, 18, 2048, 1, 1, 0, 1, True),    # stage-4 conv3
]


# kernel scheduling variants: default heuristic; few persistent CTAs (several tiles per CTA) with the default and
# with a narrow N tile
TC_MODES = {
    "default": {},
    "persistent_grid3": {"YB_CONV2D_GRID": "3"},
    "persistent_grid5_bn64": {"YB_CONV2D_GRID": "5", "YB_CONV2D_BN": "64"},
    # CTA pairs (cluster of 2 sharing the weight tile by TMA multicast): default grid, and 2 clusters walking many units
    # (odd M-tile counts -> a padding tile in the last pair)
    "pair": {"YB_CONV2D_PAIR": "1"},
    "pair_grid4_bn128": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_GRID": "4", "YB_CONV2D_BN": "128"},
    # two MMA warpgroups (each owns 64 rows of the tile), alone, persistent and with CTA pairs
    "epi2": {"YB_CONV2D_EPI": "2"},
    "epi2_grid3_bn256": {"YB_CONV2D_EPI": "2", "YB_CONV2D_GRID": "3", "YB_CONV2D_BN": "256"},
    "pair_epi2": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_EPI": "2"},
    # PDL-friendly plans (<= half an SM, weight tiles requested before griddepcontrol.wait)
    "pdl_friendly": {"YB_CONV2D_PDL": "1"},
    "pdl_friendly_bn64_grid3": {"YB_CONV2D_PDL": "1", "YB_CONV2D_BN": "64", "YB_CONV2D_GRID": "3"},
    # stream-K: equal shares of the k-block iterations per CTA / cluster, fp32 partial tiles through a workspace; few
    # CTAs give every CTA a tail, whole units and a head
    "sk": {"YB_CONV2D_SK": "1"},
    "sk_grid5": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "5"},
    "sk_grid7_bn64": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "7", "YB_CONV2D_BN": "64"},
    "sk_pair": {"YB_CONV2D_SK": "1", "YB_CONV2D_PAIR": "1"},
    "sk_pair_grid6_epi2": {"YB_CONV2D_SK": "1", "YB_CONV2D_PAIR": "1", "YB_CONV2D_GRID": "6", "YB_CONV2D_EPI": "2"},
}
if os.environ.get("YB_TEST_NO_PAIR"):   # escape hatch while the pair kernel is being brought up
    TC_MODES = {k: v for k, v in TC_MODES.items() if not k.startswith("pair")}


@functools.lru_cache(maxsize=48)
def reference(case, seed, rounded):
    """float64 act(conv + bias + residual) of make(*case, seed) and its per-element scale, NHWC; rounded: on the
    fp16-rounded x, w and residual the single-pass modes consume."""
    B, Ci, H, W, Co, k, s, p, act, wr = case
    x, w, bias, res = make(B, Ci, H, W, Co, k, s, p, True, wr, seed=seed)
    x, w = x.numpy(), w.numpy()
    res = None if res is None else res.numpy()
    if rounded:
        x, w, res = f16(x), f16(w), f16(res)
    pre, scale = conv_f64(x, w, bias.numpy(), s, p)
    if res is not None:
        rn = res.transpose(0, 2, 3, 1).astype(np.float64)
        pre, scale = pre + rn, scale + np.abs(rn)
    return act_f64(pre, act), scale


def nhwc(y):
    return y.permute(0, 2, 3, 1).double().numpy()


@pytest.mark.parametrize("mode", sorted(TC_MODES))
@pytest.mark.parametrize("case", TC_CASES)
def test_tcgen05_matches_simt_f16_and_torch(ops, case, mode, monkeypatch):
    for k_, v_ in TC_MODES[mode].items():
        monkeypatch.setenv(k_, v_)
    B, Ci, H, W, Co, k, s, p, act, wr = case
    x, w, bias, res = make(B, Ci, H, W, Co, k, s, p, True, wr, seed=1)
    y_tc, _ = run_conv(ops, x, w, bias, res, s, p, act, 1)
    y_simt, _ = run_conv(ops, x, w, bias, res, s, p, act, 2)
    # both against float64 on the SAME fp16-rounded operands, element by element
    ref, scale = reference(case, 1, True)
    what = "%s %s" % (case, mode)
    check(nhwc(y_tc), ref, scale, "f16tc", what)
    check(nhwc(y_simt), ref, scale, "f16", what)
    # and each other: two summation orders of the same products, each within its bound
    tol = 2 * K_BOUND["f16tc"] * UNIT["f16tc"] * scale + 2 * 2.0 ** -24
    err = np.abs(nhwc(y_tc) - nhwc(y_simt))
    assert (err <= tol).all(), ("tensor cores vs SIMT fp16", worst(err, tol))


# ---- split precision (YB_PREC_F16X3): fp16 hi+lo operand pairs, three MMA passes -> fp32-equivalent results -----
SPLIT_MODES = {
    "default": {},
    "persistent_grid3": {"YB_CONV2D_GRID": "3"},
    "persistent_grid5_bn64": {"YB_CONV2D_GRID": "5", "YB_CONV2D_BN": "64"},
    "pair": {"YB_CONV2D_PAIR": "1"},
    "pair_grid4_bn128": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_GRID": "4", "YB_CONV2D_BN": "128"},
    "pair_bn256": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_BN": "256"},
    "epi2": {"YB_CONV2D_EPI": "2"},
    "pair_epi2": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_EPI": "2"},
    "sk": {"YB_CONV2D_SK": "1"},
    "sk_grid5": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "5"},
    "sk_pair": {"YB_CONV2D_SK": "1", "YB_CONV2D_PAIR": "1"},
    "sk_pair_grid6": {"YB_CONV2D_SK": "1", "YB_CONV2D_PAIR": "1", "YB_CONV2D_GRID": "6"},
    "epi2_grid3": {"YB_CONV2D_EPI": "2", "YB_CONV2D_GRID": "3"},     # two groups; 1x1 residual read from global memory
}


@pytest.mark.parametrize("mode", sorted(SPLIT_MODES))
@pytest.mark.parametrize("case", TC_CASES)
def test_tcgen05_split_matches_torch_fp32(ops, case, mode, monkeypatch):
    """The reference arithmetic is fp32 (yolact.py:564-676 under eval.py:1077-1081): the split mode is compared with
    float64 on the UNROUNDED operands, element by element, within a few units of 2^-22 of each element's scale."""
    for k_, v_ in SPLIT_MODES[mode].items():
        monkeypatch.setenv(k_, v_)
    B, Ci, H, W, Co, k, s, p, act, wr = case
    x, w, bias, res = make(B, Ci, H, W, Co, k, s, p, True, wr, seed=2)
    y, _ = run_conv(ops, x, w, bias, res, s, p, act, 3)
    ref, scale = reference(case, 2, False)
    check(nhwc(y), ref, scale, "f16x3", "%s %s" % (case, mode))


def test_tcgen05_split_small_and_large_magnitudes(ops):
    """hi + lo must hold across magnitudes: tiny weights (lo would be subnormal without the power-of-two pre-scale)
    and activations up to a few thousand."""
    x, w, bias, _ = make(1, 128, 20, 20, 64, 3, 1, 1)
    for xs, ws in ((1.0, 1e-3), (3e3, 1.0), (1e-2, 1e-2), (30.0, 20.0)):
        y, _ = run_conv(ops, x * xs, w * ws, bias, None, 1, 1, 0, 3)
        ref = ref_conv(x * xs, w * ws, bias, None, 1, 1, 0)
        err = (y - ref).abs().max().item() / max(1e-30, ref.abs().max().item())
        assert err < 2e-5, (xs, ws, err)


def test_tcgen05_throughput_smoke(ops):
    # the dominant backbone shape at batch 8: 256->256 3x3 @35x35 (not a bench number; sanity only)
    x, w, bias, _ = make(8, 256, 35, 35, 256, 3, 1, 1)
    _, ms = run_conv(ops, x, w, bias, None, 1, 1, 1, 1, iters=20)
    flops = 2.0 * 8 * 35 * 35 * 256 * 256 * 9
    print("tc 3x3 256->256 @35^2 B=8: %.3f ms, %.1f TFLOP/s" % (ms, flops / ms / 1e9))
    assert ms > 0
    _, ms3 = run_conv(ops, x, w, bias, None, 1, 1, 1, 3, iters=20)
    print("split tc 3x3 256->256 @35^2 B=8: %.3f ms, %.1f algorithmic TFLOP/s (3 MMA passes)" % (ms3, flops / ms3 / 1e9))
    assert ms3 > 0
