"""float64 references of the network's max pool, bilinear resample and FastMaskIoUNet, and numpy restatements of the
activation encoders the kernels read and write (common.cuh from_f32<__half> and split_f32).

The kernels' tests (tests/test_gpu_resample.py, tests/test_gpu_maskiou.py) compare against these; the CPU test
tests/test_resample_reference_host.py pins them to torch's own operators.
"""
import numpy as np

F16_MAX = 65504.0
LO_SCALE = np.float32(2048.0)          # YB_LO_SCALE: the lo plane is kept pre-scaled by 2^11
LO_INV = np.float32(2.0 ** -11)


# ---- encoders -----------------------------------------------------------------------------------------------------
def f16_encode(v):
    """from_f32<__half>: clamp to +-65504, then fp16 with round-to-nearest-even."""
    return np.clip(np.asarray(v, np.float32), -F16_MAX, F16_MAX).astype(np.float16)


def split_encode(v):
    """split_f32: hi = fp16(c), lo' = fp16((c - hi) * 2^11) with c = v clamped to +-65504 (the residual is taken against
    the clamped value, so a saturated element gets lo' = 0).  Returns (hi, lo') as float16 arrays."""
    c = np.clip(np.asarray(v, np.float32), -F16_MAX, F16_MAX)
    hi = c.astype(np.float16)
    lo = ((c - hi.astype(np.float32)) * LO_SCALE).astype(np.float16)
    return hi, lo


def split_decode(hi, lo):
    """split_to_f32: hi + lo' * 2^-11 in fp32 (exact for every pair split_encode produces)."""
    return hi.astype(np.float32) + lo.astype(np.float32) * LO_INV


def encode_nhwc(v, precision):
    """A float NHWC tensor in the kernels' own layout: fp32, fp16, or per pixel [hi(C) | lo'(C)] (precision "f16x3")."""
    if precision == "f32":
        return np.asarray(v, np.float32)
    if precision == "f16":
        return f16_encode(v)
    hi, lo = split_encode(v)
    return np.concatenate([hi, lo], axis=-1)


def decode_nhwc(raw, precision):
    """The values the kernels read from a tensor in their own layout, as float64."""
    if precision == "f16x3":
        C = raw.shape[-1] // 2
        return split_decode(raw[..., :C], raw[..., C:]).astype(np.float64)
    return np.asarray(raw).astype(np.float64)


# ---- max pool -----------------------------------------------------------------------------------------------------
def maxpool3x3s2_f64(x):
    """nn.MaxPool2d(3, 2, 1) of NHWC x [B, H, W, C] in float64, padding acting as -inf."""
    x = np.asarray(x, np.float64)
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = np.full((B, 2 * Ho + 1, 2 * Wo + 1, C), -np.inf)
    xp[:, 1:H + 1, 1:W + 1] = x
    y = np.full((B, Ho, Wo, C), -np.inf)
    for r in range(3):
        for s in range(3):
            y = np.maximum(y, xp[:, r:r + 2 * Ho:2, s:s + 2 * Wo:2])
    return y


# ---- bilinear resample ----------------------------------------------------------------------------------------------
def bilinear_taps(n_in, n_out):
    """One axis of ATen's upsample_bilinear2d, align_corners=False, with the geometry in fp32 as the kernel computes it
    (one rounding per operation, no FMA): s = max(scale * (o + 0.5) - 0.5, 0), scale = fp32(n_in) / fp32(n_out),
    i0 = floor(s), i1 = i0 + (i0 < n_in - 1), l1 = s - i0, l0 = 1 - l1.  Returns i0, i1 (int) and l0, l1 (float64 of
    the fp32 values)."""
    f = np.float32
    scale = f(n_in) / f(n_out)
    o = np.arange(n_out, dtype=np.float32)
    s = np.maximum((scale * (o + f(0.5))).astype(np.float32) - f(0.5), f(0))
    i0 = np.floor(s).astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    l1 = (s - i0.astype(np.float32)).astype(np.float32)
    l0 = (f(1) - l1).astype(np.float32)
    return i0, i1, l0.astype(np.float64), l1.astype(np.float64)


def bilinear_f64(x, Ho, Wo, add=None, relu=False):
    """F.interpolate(size=(Ho, Wo), mode='bilinear', align_corners=False) of NHWC x in float64 (fp32 weights as above),
    then + add, then ReLU.  Returns (y, scale) with scale = sum |lambda * p| + |add|, the magnitude the kernel's
    rounding error is proportional to."""
    x = np.asarray(x, np.float64)
    _, H, W, _ = x.shape
    h0, h1, l0h, l1h = bilinear_taps(H, Ho)
    w0, w1, l0w, l1w = bilinear_taps(W, Wo)
    lh = (l0h[None, :, None, None], l1h[None, :, None, None])
    lw = (l0w[None, None, :, None], l1w[None, None, :, None])
    y = np.zeros((x.shape[0], Ho, Wo, x.shape[3]))
    scale = np.zeros_like(y)
    for a, rows in enumerate((h0, h1)):
        for b, cols in enumerate((w0, w1)):
            t = lh[a] * lw[b] * x[:, rows][:, :, cols]
            y += t
            scale += np.abs(t)
    if add is not None:
        add = np.asarray(add, np.float64)
        y = y + add
        scale = scale + np.abs(add)
    if relu:
        y = np.maximum(y, 0)
    return y, scale


# ---- FastMaskIoUNet -------------------------------------------------------------------------------------------------
MASKIOU_LAYERS = [(3, 2)] * 5 + [(1, 1)]   # (kernel, stride), no padding, each followed by ReLU (config.py maskiou_net)
MASKIOU_MIN_SIZE = 63                      # the smallest mask side the five 3x3/2 convs accept


def maskiou_out_size(n):
    """The side of each layer's output for an n-pixel input side; None where nn.Conv2d refuses the input."""
    sizes = []
    for k, s in MASKIOU_LAYERS:
        if n < k:
            return None
        n = (n - k) // s + 1
        sizes.append(n)
    return sizes


def _conv_valid(x, w, b, stride):
    """float64 unpadded conv, NHWC x [N, H, W, Ci], OIHW w, bias b: numpy, via one window gather per tap."""
    N, H, W, Ci = x.shape
    Co, _, k, _ = w.shape
    Ho, Wo = (H - k) // stride + 1, (W - k) // stride + 1
    y = np.broadcast_to(b, (N, Ho, Wo, Co)).copy()
    for r in range(k):
        for s in range(k):
            patch = x[:, r:r + stride * (Ho - 1) + 1:stride, s:s + stride * (Wo - 1) + 1:stride]
            y += patch @ w[:, :, r, s].T
    return y


def maskiou_f64(masks, weights, biases):
    """FastMaskIoUNet on masks [n, H, W] in float64: five 3x3/2 convs and one 1x1, each followed by ReLU, then the max
    over the map.  Also the magnitude chain (the same convs on |x| with |w| and |b|, no ReLU), whose maximum bounds each
    output's accumulated rounding.  Returns (out [n, C], magnitude [n, C], pre-activations of every layer)."""
    x = np.asarray(masks, np.float64)[..., None]
    m = np.abs(x)
    pre = []
    for (k, s), w, b in zip(MASKIOU_LAYERS, weights, biases):
        w, b = np.asarray(w, np.float64), np.asarray(b, np.float64)
        z = _conv_valid(x, w, b, s)
        pre.append(z)
        x = np.maximum(z, 0)
        m = _conv_valid(m, np.abs(w), np.abs(b), s)
    return x.max(axis=(1, 2)), m.max(axis=(1, 2)), pre


def maskiou_gather(out, cls):
    """output_utils.py's gather: out[i, cls[i]]."""
    return out[np.arange(out.shape[0]), np.asarray(cls, np.int64)]
