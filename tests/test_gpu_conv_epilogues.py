"""The convolution paths only the network reaches, through yb_conv2d_ex, element by element against float64:

  a. residual added AFTER the activation (Darknet blocks): the staged (TMA) epilogue, the direct epilogue and the
     CUDA-core kernels, with residuals chosen so that act-then-add and add-then-act disagree on most elements;
  b. the fused prediction head: one launch routes each output channel to the loc, conf or mask tensor (tanh on the
     mask coefficients only), written into a slice of a larger [B, P_total, width] tensor between guard bands;
  c. fp32 outputs of the half-precision kernels (DCN's conv_offset_mask), dense and into wider pixels;
  d. zero-padded output channels (Darknet's 32-channel layers written as 64-channel pixels), which must read back as
     +0 in both planes from an output buffer filled with NaN first;
  e. the tensor-core stem: one-hot "tap probe" weights that make every output channel one element of the patch (exactly
     known), and the layer shapes the network runs with the three input transforms' value ranges.

Every element is judged against the per-element float64 bound of tests/conv_reference.py.
"""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.conv_reference import (ACT_LEAKY, ACT_NONE, ACT_RELU, ACT_TANH, K_BOUND, ROUNDED, UNIT, act_f64, check,
                                  conv_ex, conv_f64, decode, f16, hd, he, out_hw, report_ratios, set_mode)  # noqa: F401
from yolact_b200 import _lib

pytestmark = pytest.mark.gpu

# tiling switches of the op-level hooks; stream-K only changes plans with the staged epilogue
MODES = {
    "default": {},
    "bn64": {"YB_CONV2D_BN": "64"},
    "bn128": {"YB_CONV2D_BN": "128"},
    "bn256": {"YB_CONV2D_BN": "256"},
    "epi2": {"YB_CONV2D_EPI": "2"},
    "pair": {"YB_CONV2D_PAIR": "1"},
    "sk": {"YB_CONV2D_SK": "1"},
    "sk_grid5": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "5"},
}
HEAD_MODES = {"default": {}, "bn32": {"YB_CONV2D_BN": "32"}, "bn64": {"YB_CONV2D_BN": "64"},
              "bn128": {"YB_CONV2D_BN": "128"}, "bn256": {"YB_CONV2D_BN": "256"}, "epi2": {"YB_CONV2D_EPI": "2"}}


def guarded(a, guard=1 << 16):
    """A device copy of `a` (fp32) between two bands of `guard` NaNs: a read outside the tensor poisons the output."""
    buf = torch.full((a.size + 2 * guard,), float("nan"), device="cuda")
    buf[guard:guard + a.size] = torch.from_numpy(np.ascontiguousarray(a, np.float32).ravel()).cuda()
    return buf[guard:guard + a.size].view(a.shape)


# ----------------------------------------------------------------------------------------------------------------
# a. residual after the activation: Darknet block conv2, 3x3 C/2 -> C, y = leaky(conv + b) + x
# ----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def darknet_block(C, H, Co=None, B=2):
    """Inputs of one Darknet block conv2, and the float64 conv of them.  The first stage's 32-channel input arrives
    zero-padded to 64 channels (its conv1 writes 64-channel pixels), with weights over the 32 real ones.  The residual
    has the opposite sign of the conv and 0.3..1.7 times its magnitude, so that leaky(v) + r and leaky(v + r) differ."""
    r = np.random.RandomState(C + H)
    Co = Co or C
    Ci = max(C // 2, 1)
    CiP = max(Ci, 64)
    x = np.zeros((B, CiP, H, H), np.float32)
    x[:, :Ci] = r.standard_normal((B, Ci, H, H))
    w = he(r, (Co, Ci, 3, 3), 9 * Ci)
    bias = (r.standard_normal(Co) * 0.1).astype(np.float32)
    pre, _ = conv_f64(x[:, :Ci], w, bias, 1, 1)
    res = (-pre * r.uniform(0.3, 1.7, pre.shape)).transpose(0, 3, 1, 2).astype(np.float32)
    return x, w, bias, res, CiP


@functools.lru_cache(maxsize=8)
def residual_reference(C, H, Co, rounded):
    x, w, bias, res, CiP = darknet_block(C, H, Co)
    Ci = w.shape[1]
    xs, ws, rs = (f16(x), f16(w), f16(res)) if rounded else (x, w, res)
    pre, scale = conv_f64(xs[:, :Ci], ws, bias, 1, 1)
    rn = rs.transpose(0, 2, 3, 1).astype(np.float64)
    after = act_f64(pre, ACT_LEAKY) + rn
    before = act_f64(pre + rn, ACT_LEAKY)
    return after, before, scale + np.abs(rn)


def run_residual_after(hd, C, H, precision, Co=None, y_f32=False):
    x, w, bias, res, CiP = darknet_block(C, H, Co)
    Co = w.shape[0]
    o = _lib.YbConvOpts()
    o.res_after_act, o.cin_pad, o.y_f32 = 1, CiP, int(y_f32)
    y = decode(conv_ex(hd, x, w, bias, res, 1, 1, ACT_LEAKY, precision, o), "f32" if y_f32 else precision, Co)
    after, before, scale = residual_reference(C, H, Co, precision in ROUNDED)
    # the residual is chosen so that the two orders disagree, beyond the tolerance, on most elements
    tol = K_BOUND[precision] * UNIT[precision] * scale
    assert (np.abs(after - before) > 10 * tol).mean() > 0.25
    check(y, after, scale, precision, "residual-after C=%d %dx%d%s" % (C, H, H, " y_f32" if y_f32 else ""))


# (C, H): the Darknet-53 stages at the 160 and 320 input sizes
DARKNET_STAGES = [(64 << s, size >> (s + 1)) for size in (160, 320) for s in range(5)]


@pytest.mark.parametrize("precision", ["f16tc", "f16x3", "f32", "f16"])
@pytest.mark.parametrize("C,H", DARKNET_STAGES, ids=lambda v: str(v))
def test_residual_after_activation_darknet_stages(hd, C, H, precision):
    run_residual_after(hd, C, H, precision)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("C,H", [(64, 80), (256, 20), (1024, 5), (1024, 10)], ids=lambda v: str(v))
def test_residual_after_activation_tilings(hd, C, H, precision, mode, monkeypatch):
    set_mode(monkeypatch, MODES[mode])
    run_residual_after(hd, C, H, precision)


@pytest.mark.parametrize("mode", ["default", "bn64", "bn128", "epi2", "pair"])
@pytest.mark.parametrize("precision,Co,y_f32", [("f16x3", 72, False), ("f16x3", 136, False), ("f16tc", 128, True),
                                                ("f16x3", 128, True)],
                         ids=["f16x3-Co72", "f16x3-Co136", "f16tc-y_f32", "f16x3-y_f32"])
def test_residual_after_activation_direct_epilogue(hd, precision, Co, y_f32, mode, monkeypatch):
    """Split outputs with Cout % 64 != 0, and fp32 outputs, go through the direct (register) epilogue."""
    set_mode(monkeypatch, MODES[mode])
    run_residual_after(hd, 128, 20, precision, Co=Co, y_f32=y_f32)


def test_residual_after_relu_refused_by_the_staged_epilogue_only(hd):
    """The staged epilogue has an act-then-add instance for LeakyReLU only: ReLU there is refused instead of silently
    adding before the activation; the direct epilogue (fp32 output) and the CUDA-core kernel compute it."""
    x, w, bias, res, _ = darknet_block(128, 20)
    o = _lib.YbConvOpts()
    o.res_after_act = 1
    with pytest.raises(_lib.YbError, match="residual after the activation needs LeakyReLU"):
        conv_ex(hd, x, w, bias, res, 1, 1, ACT_RELU, "f16tc", o)
    for precision, y_f32 in (("f16tc", 1), ("f16x3", 1), ("f32", 0)):
        o = _lib.YbConvOpts()
        o.res_after_act, o.y_f32 = 1, y_f32
        y = decode(conv_ex(hd, x, w, bias, res, 1, 1, ACT_RELU, precision, o), "f32", 128)
        xs, ws, rs = (f16(x), f16(w), f16(res)) if precision in ROUNDED else (x, w, res)
        pre, scale = conv_f64(xs, ws, bias, 1, 1)
        rn = rs.transpose(0, 2, 3, 1).astype(np.float64)
        check(y, act_f64(pre, ACT_RELU) + rn, scale + np.abs(rn), precision, "residual after relu")


# ----------------------------------------------------------------------------------------------------------------
# b. the fused prediction head: Cin 256 -> A * (4 + 81 + 32), three segments with their own strides
# ----------------------------------------------------------------------------------------------------------------
NC, MD = 81, 32
GUARD_BEFORE, GUARD_AFTER = 5, 300      # priors; after >= Cout / 4 elements of the narrowest tensor
SENTINEL = -12345.0


@functools.lru_cache(maxsize=2)
def head_case(A, S, B):
    r = np.random.RandomState(100 * A + 10 * S + B)
    Co = A * (4 + NC + MD)
    x = np.maximum(r.standard_normal((B, 256, S, S)), 0).astype(np.float32)   # the upfeature layer's ReLU output
    w = he(r, (Co, 256, 3, 3), 9 * 256 / 2)
    bias = (r.standard_normal(Co) * 0.5).astype(np.float32)
    y, scale = conv_f64(x, w, bias, 1, 1)
    y16 = F.conv2d(torch.from_numpy(f16(x)).double(), torch.from_numpy(f16(w)).double(),
                   torch.from_numpy(bias).double(), padding=1).permute(0, 2, 3, 1).numpy()
    return x, w, bias, {False: (y, scale), True: (y16, scale)}   # the scale of the rounded operands differs by 2^-11


def run_head(hd, A, S, B, precision, gaps=False):
    """One level's head into slices of [B, P_total, width] tensors, whose other priors are a guard band of SENTINEL;
    the slice itself starts as NaN.  gaps: each segment leaves out its first channel (stored nowhere)."""
    x, w, bias, ref = head_case(A, S, B)
    widths = (4, NC, MD)
    P = S * S * A
    P_total = GUARD_BEFORE + P + GUARD_AFTER
    bufs = []
    o = _lib.YbConvOpts()
    o.nseg = 3
    begin = 0
    for i, width in enumerate(widths):
        buf = torch.full((B, P_total, width), SENTINEL, device="cuda")
        buf[:, GUARD_BEFORE:GUARD_BEFORE + P] = float("nan")
        bufs.append(buf)
        o.seg_begin[i] = begin + (1 if gaps else 0)
        o.seg_end[i] = begin + A * width
        begin += A * width
        o.seg_act[i] = ACT_TANH if i == 2 else ACT_NONE
        o.seg_pix_stride[i] = A * width
        o.seg_batch_stride[i] = P_total * width
        o.seg_y[i] = buf[0, GUARD_BEFORE].data_ptr()
    conv_ex(hd, x, w, bias, None, 1, 1, ACT_NONE, precision, o)
    pre, scale = ref[precision in ROUNDED]
    for i, (buf, width) in enumerate(zip(bufs, widths)):
        got = buf.cpu().numpy().astype(np.float64)
        guard = np.ones(P_total, bool)
        guard[GUARD_BEFORE:GUARD_BEFORE + P] = False
        assert (got[:, guard] == SENTINEL).all(), "segment %d wrote outside its slice" % i
        got = got[:, ~guard].reshape(B, S, S, A * width)
        lo, hi = o.seg_begin[i], o.seg_end[i]
        want, sc = pre[..., lo:hi], scale[..., lo:hi]
        if i == 2:
            want = np.tanh(want)
        if gaps:   # column j holds channel seg_begin + j: the last column of every pixel keeps its NaN
            assert np.isnan(got[..., -1]).all(), "segment %d stored a channel outside [seg_begin, seg_end)" % i
            got = got[..., :-1]
        # the bound carries over through tanh (|tanh'| <= 1); + 2^-22 for tanhf itself
        tol_extra = 2.0 ** -22 if i == 2 else 0.0
        check(got, want, sc + tol_extra / (K_BOUND[precision] * UNIT[precision]), precision,
              "head A=%d %dx%d B=%d %s" % (A, S, S, B, ("loc", "conf", "mask")[i]))


HEAD_LEVELS = [(69, 1), (35, 1), (35, 3), (18, 3), (9, 3), (5, 1), (5, 3), (3, 3), (2, 1), (1, 3)]   # (S, B)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("A", [3, 9])
@pytest.mark.parametrize("S,B", HEAD_LEVELS, ids=lambda v: str(v))
def test_fused_head_levels(hd, S, B, A, precision):
    run_head(hd, A, S, B, precision)


@pytest.mark.parametrize("mode", sorted(HEAD_MODES))
@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("A", [3, 9])
@pytest.mark.parametrize("S,B", [(18, 3), (5, 1)], ids=lambda v: str(v))
def test_fused_head_tilings(hd, S, B, A, precision, mode, monkeypatch):
    """The segment boundaries (channels 12 and 255; 36 and 765 for A = 9) fall inside an 8-column fragment group and
    inside an N tile for every N tile width."""
    set_mode(monkeypatch, HEAD_MODES[mode])
    run_head(hd, A, S, B, precision)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("mode", ["default", "bn32"])
def test_fused_head_channels_outside_every_segment_are_not_stored(hd, precision, mode, monkeypatch):
    set_mode(monkeypatch, HEAD_MODES[mode])
    run_head(hd, 3, 5, 3, precision, gaps=True)


# ----------------------------------------------------------------------------------------------------------------
# c. fp32 output from the half-precision kernels: conv_offset_mask, 3x3 -> 27 (YOLACT++ DCN layers)
# ----------------------------------------------------------------------------------------------------------------
OFFSET_CONVS = [(128, 69, 1), (128, 138, 2), (256, 35, 1), (256, 69, 2), (512, 18, 1), (512, 35, 2)]   # Cin, H, stride


@pytest.mark.parametrize("pix_stride", [0, 32], ids=["dense", "pixel-stride-32"])
@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("Cin,H,stride", OFFSET_CONVS, ids=lambda v: str(v))
def test_fp32_output_conv_offset_mask(hd, Cin, H, stride, precision, pix_stride):
    r = np.random.RandomState(Cin + H)
    B = 2
    x = r.standard_normal((B, Cin, H, H)).astype(np.float32)
    w = he(r, (27, Cin, 3, 3), 9 * Cin)
    bias = (r.standard_normal(27) * 0.1).astype(np.float32)
    o = _lib.YbConvOpts()
    o.y_f32, o.y_pix_stride = 1, pix_stride
    raw = conv_ex(hd, x, w, bias, None, stride, 1, ACT_NONE, precision, o)
    if pix_stride:   # the pixels' tails are not written
        assert torch.isnan(raw[..., 27:]).all()
    xs, ws = (f16(x), f16(w)) if precision in ROUNDED else (x, w)
    ref, scale = conv_f64(xs, ws, bias, stride, 1)
    check(decode(raw, "f32", 27), ref, scale, precision, "offset conv Cin=%d %dx%d s%d" % (Cin, H, H, stride))


# ----------------------------------------------------------------------------------------------------------------
# d. zero-padded output channels: Darknet block conv1 (1x1 64 -> 32, written as 64) and the Darknet stem (cpad 64)
# ----------------------------------------------------------------------------------------------------------------
def check_pad_channels(raw, precision, Co, Cp):
    """Every pad channel, in both planes, is +0 (bit pattern 0) in a buffer that held NaN."""
    bits = raw.view(torch.int16)
    planes = [bits[..., Co:Cp]] + ([bits[..., Cp + Co:2 * Cp]] if precision == "f16x3" else [])
    for pl in planes:
        assert (pl == 0).all(), "%d pad elements are not +0" % (pl != 0).sum().item()


@pytest.mark.parametrize("mode", ["default", "bn128", "epi2", "pair", "sk"])
@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("B,H,W", [(2, 80, 80), (1, 41, 37), (3, 5, 5)], ids=lambda v: str(v))
def test_zero_padded_output_channels_darknet_conv1(hd, B, H, W, precision, mode, monkeypatch):
    set_mode(monkeypatch, MODES[mode])
    r = np.random.RandomState(H * W)
    x = r.standard_normal((B, 64, H, W)).astype(np.float32)
    w = he(r, (32, 64, 1, 1), 64)
    bias = (r.standard_normal(32) * 0.1).astype(np.float32)
    o = _lib.YbConvOpts()
    o.cout_pad = 64
    raw = conv_ex(hd, x, w, bias, None, 1, 0, ACT_LEAKY, precision, o)
    check_pad_channels(raw, precision, 32, 64)
    xs, ws = (f16(x), f16(w)) if precision in ROUNDED else (x, w)
    ref, scale = conv_f64(xs, ws, bias, 1, 0)
    check(decode(raw, precision, 64)[..., :32], act_f64(ref, ACT_LEAKY), scale, precision, "conv1 %dx%d" % (H, W))


# ----------------------------------------------------------------------------------------------------------------
# e. the tensor-core stem: 7x7/2 pad 3 3 -> 64 ReLU (ResNet), 3x3/1 pad 1 3 -> 32 LeakyReLU (Darknet)
# ----------------------------------------------------------------------------------------------------------------
STEMS = {"7x7": (7, 2, 3, 64, ACT_RELU), "3x3": (3, 1, 1, 32, ACT_LEAKY)}


def stem_input(r, B, H, W, rng):
    """The value ranges of the three input transforms: normalize (about +-2.7), subtract_means (-124..152), none
    (0..255: the hi / lo split carries low bits)."""
    if rng == "normalize":
        return np.clip(r.standard_normal((B, 3, H, W)), -2.7, 2.7).astype(np.float32)
    if rng == "subtract_means":
        return (r.uniform(0, 255, (B, 3, H, W)) - np.array([123.68, 116.78, 103.94])[None, :, None, None]).astype(np.float32)
    return r.uniform(0, 255, (B, 3, H, W)).astype(np.float32)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("B,H,W", [(2, 13, 11), (2, 23, 24), (1, 1, 1)], ids=lambda v: str(v))
@pytest.mark.parametrize("stem", sorted(STEMS))
def test_stem_tap_probe(hd, stem, B, H, W, precision):
    """One-hot weights, no bias, no activation: output channel o selects patch element k = c*KS^2 + r*KS + s, so the
    output is x at one tap (0 in the padding) -- fp16(x) exactly in f16tc, x to within 2^-22 in f16x3 -- at every
    border and corner.  Channels past K (and the zero tail of the padded K) must add nothing: they read exactly 0."""
    ks, stride, pad, Co, _ = STEMS[stem]
    K = 3 * ks * ks
    r = np.random.RandomState(H * W + ks)
    x = stem_input(r, B, H, W, "subtract_means")
    xd = guarded(x)
    Ho, Wo = out_hw(H, W, ks, stride, pad)
    xp = np.pad(x.astype(np.float64), ((0, 0), (0, 0), (pad, pad + ks), (pad, pad + ks)))
    for k0 in range(0, K, Co):           # 147 taps: three runs of 64 channels
        w = np.zeros((Co, 3, ks, ks), np.float32)
        want = np.zeros((B, Ho, Wo, Co))
        for o in range(Co):
            k = k0 + o
            if k >= K:
                continue
            c, rr, s = k // (ks * ks), k % (ks * ks) // ks, k % ks
            w[o, c, rr, s] = 1.0
            want[..., o] = xp[:, c, rr:rr + stride * Ho:stride, s:s + stride * Wo:stride][:, :Ho, :Wo]
        y = decode(conv_ex(hd, xd, w, None, None, stride, pad, ACT_NONE, precision), precision, Co)
        if precision == "f16tc":
            exact = want.astype(np.float16).astype(np.float64)
            bad = ~(y == exact)
        else:
            bad = ~(np.abs(y - want) <= 2.0 ** -22 * np.abs(want))
        if bad.any():
            b, ho, wo, o = np.argwhere(bad)[0]
            pytest.fail("%d probe outputs wrong; first: image %d pixel (%d, %d) channel %d (k = %d): got %r want %r"
                        % (bad.sum(), b, ho, wo, o, k0 + o, y[b, ho, wo, o], want[b, ho, wo, o]))


STEM_SHAPES = {   # (B, H, W) per stem: M = B * Ho * Wo = 1, 127, 128, 129; odd and even sizes
    "7x7": [(1, 1, 1), (1, 253, 1), (2, 15, 16), (3, 85, 2)],
    "3x3": [(1, 1, 1), (1, 127, 1), (2, 8, 8), (3, 43, 1)],
}


@functools.lru_cache(maxsize=2)
def stem_case(stem, B, H, W, rng, wscale):
    ks, stride, pad, Co, act = STEMS[stem]
    r = np.random.RandomState(B * H * W + ks)
    x = stem_input(r, B, H, W, rng)
    w = he(r, (Co, 3, ks, ks), 3 * ks * ks) * np.float32(wscale)
    bias = (r.standard_normal(Co) * 0.1 * wscale).astype(np.float32)
    return x, w, bias, {rd: conv_f64(*((f16(x), f16(w)) if rd else (x, w)), bias, stride, pad) for rd in (False, True)}


def run_stem(hd, stem, B, H, W, rng, precision, wscale=1.0, cpad=0):
    ks, stride, pad, Co, act = STEMS[stem]
    x, w, bias, ref = stem_case(stem, B, H, W, rng, wscale)
    o = _lib.YbConvOpts()
    o.cout_pad = cpad
    Cp = max(Co, cpad)
    raw = conv_ex(hd, guarded(x), w, bias, None, stride, pad, act, precision, o)
    if cpad:
        check_pad_channels(raw, precision, Co, Cp)
    pre, scale = ref[precision in ROUNDED]
    check(decode(raw, precision, Cp)[..., :Co], act_f64(pre, act), scale, precision,
          "stem %s %dx%dx%d %s w*%g" % (stem, B, H, W, rng, wscale))


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("rng", ["normalize", "subtract_means", "none"])
@pytest.mark.parametrize("stem,B,H,W", [(s, *shape) for s in sorted(STEMS) for shape in STEM_SHAPES[s]],
                         ids=lambda v: str(v))
def test_stem_layer_shapes_tile_edges(hd, stem, B, H, W, rng, precision):
    run_stem(hd, stem, B, H, W, rng, precision)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("stem,B,H,W,rng", [("7x7", 1, 550, 550, "normalize"), ("7x7", 2, 700, 700, "subtract_means"),
                                            ("3x3", 1, 550, 550, "none"), ("3x3", 1, 700, 700, "normalize")],
                         ids=lambda v: str(v))
def test_stem_network_sizes(hd, stem, B, H, W, rng, precision):
    run_stem(hd, stem, B, H, W, rng, precision)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("stem", sorted(STEMS))
def test_stem_tiny_weights(hd, stem, precision):
    """Weights of 1e-3: the split mode's power-of-two pre-scale keeps the lo halves normal."""
    run_stem(hd, stem, 2, 37, 29, "none", precision, wscale=1e-3)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("B,H,W", [(2, 160, 160), (1, 37, 29)], ids=lambda v: str(v))
def test_zero_padded_output_channels_darknet_stem(hd, B, H, W, precision):
    run_stem(hd, "3x3", B, H, W, "normalize", precision, cpad=64)
