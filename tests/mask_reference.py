"""Float64 reference of mask assembly (yb_postprocess: proto @ coef^T -> sigmoid -> crop -> bilinear -> > 0.5) with a
per-pixel error bound, so that a kernel's binary mask can be judged pixel by pixel.

The geometry follows the reference exactly, in fp32: sanitize_coordinates and the crop comparisons (box_utils.py:327-373,
NaN propagating as torch.min / torch.max / clamp do), scale = f32(in) / f32(out), and ATen's align_corners=False source
index and lambdas (O.bilinear_resize).  The values run in float64: the lincomb, the sigmoid, the crop multiply and the
bilinear blend.

Each pixel gets its float64 value v and a bound e on how far the kernel's fp32 value can be from v: the bilinear blend
of the per-source bound 0.25 (k + 2) u sum_j |p_j c_j| + 4 u (the fmaf chain through the sigmoid's slope <= 1/4, then
expf and the division), plus 8 u for the fp32 blend, u = 2^-24.  A pixel is decided when |v - 0.5| > 2 e: the kernel's
bit must then equal v > 0.5.  The few pixels closer to 0.5 are left out of the comparison."""
import numpy as np

from oracle import yolact_oracle as O

U24 = 2.0 ** -24
f32 = np.float32


def crop_windows(box, ph, pw, crop=True):
    """fp32 crop windows (x1, x2, y1, y2) [n] in prototype coordinates: sanitize_coordinates with padding 1; the whole
    map without crop."""
    box = np.asarray(box, f32).reshape(-1, 4)
    n = box.shape[0]
    if not crop:
        z = np.zeros(n, f32)
        return z, np.full(n, pw, f32), z, np.full(n, ph, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        x1, x2 = O.sanitize_coordinates(box[:, 0], box[:, 2], pw, 1)
        y1, y2 = O.sanitize_coordinates(box[:, 1], box[:, 3], ph, 1)
    return x1, x2, y1, y2


def crop_keep(box, ph, pw, crop=True):
    """[n, ph, pw] bool: the prototype positions box_utils.crop keeps (every comparison with NaN is false)."""
    x1, x2, y1, y2 = crop_windows(box, ph, pw, crop)
    c = np.arange(pw, dtype=f32)[None, :]
    r = np.arange(ph, dtype=f32)[None, :]
    with np.errstate(invalid="ignore"):
        cols = (c >= x1[:, None]) & (c < x2[:, None])
        rows = (r >= y1[:, None]) & (r < y2[:, None])
    return rows[:, :, None] & cols[:, None, :]


def interp_table(out, inn):
    """ATen upsample_bilinear2d, align_corners=False, fp32: source indices i0, i1 and lambdas l0, l1 per output index."""
    scale = f32(inn) / f32(out)
    d = np.arange(out, dtype=f32)
    s = np.maximum(scale * (d + f32(0.5)) - f32(0.5), f32(0)).astype(f32)
    i0 = np.minimum(s.astype(np.int64), inn - 1)
    i1 = i0 + (i0 < inn - 1)
    l1 = (s - i0.astype(f32)).astype(f32)
    return i0, i1, (f32(1) - l1).astype(f32), l1


def proto_reference(proto, coef, box, crop=True):
    """Cropped sigmoid masks at prototype resolution: (value [n, ph, pw] float64, bound [n, ph, pw], keep [n, ph, pw]).
    Outside the crop window value and bound are 0: the kernels store an exact zero there."""
    proto = np.asarray(proto, f32)
    coef = np.asarray(coef, f32).reshape(-1, proto.shape[2])
    ph, pw, k = proto.shape
    n = coef.shape[0]
    p = proto.reshape(-1, k).astype(np.float64)
    c = coef.astype(np.float64)
    lin = (p @ c.T).T.reshape(n, ph, pw)
    mag = (np.abs(p) @ np.abs(c).T).T.reshape(n, ph, pw)
    with np.errstate(over="ignore"):
        sig = 1.0 / (1.0 + np.exp(-lin))
    keep = crop_keep(box, ph, pw, crop)
    value = np.where(keep, sig, 0.0)
    bound = np.where(keep, 0.25 * (k + 2) * U24 * mag + 4 * U24, 0.0)
    return value, bound, keep


def mask_reference(proto, coef, box, out_h, out_w, crop=True):
    """(v, e) [n, out_h, out_w] float64: the bilinear value of every output pixel and its error bound."""
    value, bound, _ = proto_reference(proto, coef, box, crop)
    _, ph, pw = value.shape
    h0, h1, lh0, lh1 = interp_table(out_h, ph)
    w0, w1, lw0, lw1 = interp_table(out_w, pw)
    lh0, lh1, lw0, lw1 = (a.astype(np.float64) for a in (lh0, lh1, lw0, lw1))

    def blend(x):   # columns first, then rows: the same linear blend as top / bot / out, in float64
        t = x[:, :, w0] * lw0 + x[:, :, w1] * lw1
        return t[:, h0, :] * lh0[:, None] + t[:, h1, :] * lh1[:, None]

    return blend(value), blend(bound) + 8 * U24


def decide(v, e):
    """(decided, want): the pixels whose bit the bound fixes, and the bit v > 0.5."""
    return np.abs(v - 0.5) > 2 * e, v > 0.5
