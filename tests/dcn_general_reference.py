"""float64 restatements of the dcn_v2 drop-in's general forward ops, which the GPU tests judge the kernels against
(checked on the CPU by tests/test_dcn_general_reference_host.py).

dcn_columns   modulated_deformable_im2col_gpu_kernel (external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:125-195) for any
              kernel size, per-axis stride / padding / dilation and deformable groups -- oracle.dcn_v2_columns
              generalised: the same fp32 positions, floors and fractional weights, the blend in `acc`.
psroi_pool    DeformablePSROIPoolForwardKernel (external/DCNv2/src/cuda/dcn_v2_psroi_pooling_cuda.cu:59-146): the RoI,
              bin, part and sample geometry in fp32, one operation at a time in the source's order, the blend, the sum
              and the mean in `acc`.
"""
import numpy as np

f32 = np.float32


def out_size(n, k, stride, pad, dil):
    return (n + 2 * pad - (dil * (k - 1) + 1)) // stride + 1


def dcn_columns(x, offset, mask, kernel, stride, pad, dil, dg, acc=np.float64, with_abs=False):
    """x [B,C,H,W], offset [B,2*dg*kh*kw,Ho,Wo], mask [B,dg*kh*kw,Ho,Wo]; kernel, stride, pad, dil are (h, w) pairs ->
    columns [B,C,kh*kw,Ho,Wo] of dtype acc (and, with_abs, the sum over corners of |weight * mask * x|)."""
    x = np.asarray(x, f32)
    offset = np.asarray(offset, f32)
    mask = np.asarray(mask, f32)
    B, C, H, W = x.shape
    kh, kw = kernel
    taps = kh * kw
    Ho, Wo = offset.shape[2:]
    cg = C // dg
    cols = np.zeros((B, C, taps, Ho, Wo), acc)
    mag = np.zeros((B, C, taps, Ho, Wo), acc) if with_abs else None
    zero = acc(0)
    ho = np.arange(Ho)[:, None]
    wo = np.arange(Wo)[None, :]
    for g in range(dg):
        xs = x[:, g * cg:(g + 1) * cg]
        for t in range(taps):
            i, j = divmod(t, kw)
            # dcn_v2_im2col_cuda.cu:177-178: int base + fp32 offset, one fp32 rounding
            h_im = (f32(1) * (ho * stride[0] - pad[0] + i * dil[0]) + offset[:, g * 2 * taps + 2 * t]).astype(f32)
            w_im = (f32(1) * (wo * stride[1] - pad[1] + j * dil[1]) + offset[:, g * 2 * taps + 2 * t + 1]).astype(f32)
            with np.errstate(invalid="ignore"):
                ok = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)                     # [B,Ho,Wo]
            h = np.where(ok, h_im, f32(0))
            w = np.where(ok, w_im, f32(0))
            hl = np.floor(h).astype(np.int64)
            wl = np.floor(w).astype(np.int64)
            hh, wh = hl + 1, wl + 1
            lh = (h - hl).astype(f32)
            lw = (w - wl).astype(f32)
            uh, uw = (1 - lh).astype(f32), (1 - lw).astype(f32)
            lh, lw, uh, uw = (a.astype(acc)[:, None] for a in (lh, lw, uh, uw))
            bidx = np.arange(B)[:, None, None, None]
            cidx = np.arange(cg)[None, :, None, None]

            def corner(hi, wi, exists):
                v = xs[bidx, cidx, np.clip(hi, 0, H - 1)[:, None], np.clip(wi, 0, W - 1)[:, None]].astype(acc)
                return np.where((exists & ok)[:, None], v, zero)

            t1 = (uh * uw) * corner(hl, wl, (hl >= 0) & (wl >= 0))
            t2 = (uh * lw) * corner(hl, wh, (hl >= 0) & (wh <= W - 1))
            t3 = (lh * uw) * corner(hh, wl, (hh <= H - 1) & (wl >= 0))
            t4 = (lh * lw) * corner(hh, wh, (hh <= H - 1) & (wh <= W - 1))
            m = mask[:, g * taps + t].astype(acc)[:, None]
            cols[:, g * cg:(g + 1) * cg, t] = np.where(ok[:, None], t1 + t2 + t3 + t4, zero) * m
            if with_abs:
                mag[:, g * cg:(g + 1) * cg, t] = np.where(ok[:, None], abs(t1) + abs(t2) + abs(t3) + abs(t4), zero) * abs(m)
    return (cols, mag) if with_abs else cols


def dcn_contract(cols, weight, bias, acc=np.float64):
    """columns [B,C,taps,Ho,Wo] x weight [Co,C,kh,kw] + bias [Co] -> [B,Co,Ho,Wo] (dcn_v2_cuda.cu:123-163)."""
    B, C, taps, Ho, Wo = cols.shape
    Co = weight.shape[0]
    wm = np.asarray(weight, f32).reshape(Co, C * taps).astype(acc)
    out = np.einsum("ok,bkp->bop", wm, cols.reshape(B, C * taps, Ho * Wo).astype(acc))
    if bias is not None:
        out = out + np.asarray(bias, f32).astype(acc)[None, :, None]
    return out.reshape(B, Co, Ho, Wo)


def dcn_forward(x, offset, mask, weight, bias, stride, pad, dil, dg):
    """float64 output and the per-element scale sum_k |w_k| * mag_k + |bias| its rounding error is proportional to."""
    kernel = weight.shape[2:]
    cols, mag = dcn_columns(x, offset, mask, kernel, stride, pad, dil, dg, with_abs=True)
    ref = dcn_contract(cols, weight, bias)
    scale = dcn_contract(mag, np.abs(weight), None if bias is None else np.abs(bias))
    return ref, scale


def round_half_away(v):
    """C's round() of fp32 values (half away from zero); exact in float64."""
    v64 = np.asarray(v, f32).astype(np.float64)
    return np.copysign(np.floor(np.abs(v64) + 0.5), v64).astype(f32)


def psroi_geometry(rois, trans, R, output_dim, spatial_scale, group_size, pooled, part_size, spp, trans_std, no_trans,
                   num_classes):
    """fp32 per-output-element geometry [R, output_dim, pooled, pooled]: batch index, input channel, wstart, hstart,
    sub-bin sizes."""
    rois = np.asarray(rois, f32).reshape(-1, 5)
    P = pooled
    n = np.arange(R)[:, None, None, None]
    ctop = np.arange(output_dim)[None, :, None, None]
    ph = np.arange(P)[None, None, :, None]
    pw = np.arange(P)[None, None, None, :]
    s = f32(spatial_scale)
    rs_w = (round_half_away(rois[:, 1]) * s - f32(0.5)).astype(f32)
    rs_h = (round_half_away(rois[:, 2]) * s - f32(0.5)).astype(f32)
    re_w = ((round_half_away(rois[:, 3]) + f32(1)) * s - f32(0.5)).astype(f32)
    re_h = ((round_half_away(rois[:, 4]) + f32(1)) * s - f32(0.5)).astype(f32)
    roi_w = np.maximum(re_w - rs_w, f32(0.1)).astype(f32)
    roi_h = np.maximum(re_h - rs_h, f32(0.1)).astype(f32)
    bin_w, bin_h = roi_w / f32(P), roi_h / f32(P)
    sub_w, sub_h = bin_w / f32(spp), bin_h / f32(spp)
    if no_trans:
        tx = ty = np.zeros((R, output_dim, P, P), f32)
    else:
        trans = np.asarray(trans, f32)
        part_h = np.floor((ph.astype(f32) / f32(P)) * f32(part_size)).astype(np.int64)
        part_w = np.floor((pw.astype(f32) / f32(P)) * f32(part_size)).astype(np.int64)
        cls = ctop // (output_dim // num_classes)
        tx = trans[n, 2 * cls, part_h, part_w] * f32(trans_std)
        ty = trans[n, 2 * cls + 1, part_h, part_w] * f32(trans_std)
    col = lambda a: a[:, None, None, None]
    wstart = (pw.astype(f32) * col(bin_w) + col(rs_w)).astype(f32) + (tx * col(roi_w)).astype(f32)
    hstart = (ph.astype(f32) * col(bin_h) + col(rs_h)).astype(f32) + (ty * col(roi_h)).astype(f32)
    gw = np.clip(np.floor((pw.astype(f32) * f32(group_size)) / f32(P)).astype(np.int64), 0, group_size - 1)
    gh = np.clip(np.floor((ph.astype(f32) * f32(group_size)) / f32(P)).astype(np.int64), 0, group_size - 1)
    c = (ctop * group_size + gh) * group_size + gw
    b = rois[:, 0].astype(np.int64)
    shape = (R, output_dim, P, P)
    return (np.broadcast_to(col(b), shape), np.broadcast_to(c, shape), wstart.astype(f32), hstart.astype(f32),
            np.broadcast_to(col(sub_w), shape), np.broadcast_to(col(sub_h), shape))


def psroi_pool(x, rois, trans, spatial_scale, output_dim, group_size, pooled, part_size, sample_per_part, trans_std,
               no_trans, acc=np.float64):
    """-> (output, count, mag) [R, output_dim, pooled, pooled]: the pooled values in `acc`, the samples counted, and
    (sum over the counted samples of the four |corner weight * value|) / count, the scale of the rounding error."""
    x = np.asarray(x, f32)
    N, C, H, W = x.shape
    R = np.asarray(rois).reshape(-1, 5).shape[0]
    num_classes = 1 if no_trans else np.asarray(trans).shape[1] // 2
    b, c, wstart, hstart, sub_w, sub_h = psroi_geometry(rois, trans, R, output_dim, spatial_scale, group_size, pooled,
                                                        part_size, sample_per_part, trans_std, no_trans, num_classes)
    total = np.zeros(wstart.shape, acc)
    mag = np.zeros(wstart.shape, acc)
    count = np.zeros(wstart.shape, np.int64)
    for ih in range(sample_per_part):
        for iw in range(sample_per_part):
            w = (wstart + (f32(iw) * sub_w).astype(f32)).astype(f32)
            h = (hstart + (f32(ih) * sub_h).astype(f32)).astype(f32)
            ok = ~((w < -0.5) | (w > W - 0.5) | (h < -0.5) | (h > H - 0.5))
            w = np.minimum(np.maximum(w, f32(0)), f32(W - 1))
            h = np.minimum(np.maximum(h, f32(0)), f32(H - 1))
            x1, x2 = np.floor(w).astype(np.int64), np.ceil(w).astype(np.int64)
            y1, y2 = np.floor(h).astype(np.int64), np.ceil(h).astype(np.int64)
            dx = (w - x1.astype(f32)).astype(f32)
            dy = (h - y1.astype(f32)).astype(f32)
            ux, uy = (f32(1) - dx).astype(acc), (f32(1) - dy).astype(acc)
            dx, dy = dx.astype(acc), dy.astype(acc)
            v = lambda yy, xx: x[b, c, yy, xx].astype(acc)
            terms = ((ux * uy) * v(y1, x1), (ux * dy) * v(y2, x1), (dx * uy) * v(y1, x2), (dx * dy) * v(y2, x2))
            val = ((terms[0] + terms[1]) + terms[2]) + terms[3]
            total = total + np.where(ok, val, acc(0))
            mag = mag + np.where(ok, sum(abs(t_) for t_ in terms), acc(0))
            count = count + ok
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(count > 0, total / np.maximum(count, 1).astype(acc), acc(0)).astype(acc)
        mag = np.where(count > 0, mag / np.maximum(count, 1), 0)
    return out, count, mag
