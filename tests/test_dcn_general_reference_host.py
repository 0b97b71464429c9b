"""The float64 restatements the general DCNv2 and deformable PS-RoI pooling GPU tests judge against, checked on the CPU:
the grouped, any-kernel deformable im2col against oracle.dcn_v2_columns (3x3, one group) and against
torchvision.ops.deform_conv2d in float64; the pooling restatement against a scalar fp32 brute force written from the
reference kernel separately, and against hand-derived cases."""
import numpy as np
import pytest
import torch
from torchvision.ops import deform_conv2d

from oracle import yolact_oracle as O
from tests.dcn_general_reference import dcn_columns, dcn_contract, out_size, psroi_pool

f32 = np.float32


def random_case(r, B, C, Co, H, W, kernel, stride, pad, dil, dg, off_scale=2.0):
    Ho, Wo = out_size(H, kernel[0], stride[0], pad[0], dil[0]), out_size(W, kernel[1], stride[1], pad[1], dil[1])
    taps = kernel[0] * kernel[1]
    x = r.standard_normal((B, C, H, W)).astype(f32)
    off = (r.standard_normal((B, 2 * dg * taps, Ho, Wo)) * off_scale).astype(f32)
    msk = r.uniform(size=(B, dg * taps, Ho, Wo)).astype(f32)
    w = r.standard_normal((Co, C) + tuple(kernel)).astype(f32)
    bias = r.standard_normal(Co).astype(f32)
    return x, off, msk, w, bias


GENERAL = [  # C, dg, kernel, stride, pad, dil
    (8, 1, (1, 1), (1, 1), (0, 0), (1, 1)),
    (8, 2, (1, 3), (1, 2), (0, 1), (1, 1)),
    (12, 4, (5, 5), (2, 1), (2, 3), (1, 2)),
    (8, 2, (7, 7), (1, 1), (3, 3), (1, 1)),
    (16, 4, (3, 3), (2, 3), (1, 0), (2, 1)),
    (6, 2, (3, 1), (1, 1), (1, 0), (3, 1)),
]


@pytest.mark.parametrize("C,dg,kernel,stride,pad,dil", GENERAL)
def test_grouped_columns_against_torchvision_float64(C, dg, kernel, stride, pad, dil):
    r = np.random.RandomState(C * 7 + dg + kernel[0])
    x, off, msk, w, bias = random_case(r, 2, C, 5, 11, 9, kernel, stride, pad, dil, dg)
    ref = dcn_contract(dcn_columns(x, off, msk, kernel, stride, pad, dil, dg), w, bias)
    tv = deform_conv2d(torch.from_numpy(x).double(), torch.from_numpy(off).double(), torch.from_numpy(w).double(),
                       torch.from_numpy(bias).double(), stride=stride, padding=pad, dilation=dil,
                       mask=torch.from_numpy(msk).double()).numpy()
    assert ref.shape == tv.shape
    # torchvision takes the positions in float64, the reference (and the restatement) in fp32: one fp32 rounding of
    # each position, times the slope of the bilinear surface (|x| <= ~5, |w| * |mask| summed over taps * C)
    scale = np.abs(w).reshape(w.shape[0], -1).sum(1)[None, :, None, None] * np.abs(x).max()
    assert np.all(np.abs(ref - tv) <= 2e-5 * scale), np.abs(ref - tv).max()


def test_one_group_3x3_is_the_oracle():
    r = np.random.RandomState(4)
    x, off, msk, _, _ = random_case(r, 2, 16, 3, 9, 8, (3, 3), (2, 2), (2, 2), (2, 2), 1)
    mine = dcn_columns(x, off, msk, (3, 3), (2, 2), (2, 2), (2, 2), 1, acc=np.float32)
    assert np.array_equal(mine, O.dcn_v2_columns(x, off, msk, 2, 2, 2))


def test_groups_read_their_own_offsets():
    """Group g's channels move with group g's offsets only: shifting group 1 by a whole pixel shifts its columns."""
    x = np.arange(2 * 4 * 6 * 6, dtype=f32).reshape(2, 4, 6, 6)
    off = np.zeros((2, 2 * 2 * 9, 6, 6), f32)
    off[:, 18 + 1::2] = 1.0               # group 1: every tap one column to the right
    msk = np.ones((2, 18, 6, 6), f32)
    cols = dcn_columns(x, off, msk, (3, 3), (1, 1), (1, 1), (1, 1), 2)
    base = dcn_columns(x, np.zeros_like(off), msk, (3, 3), (1, 1), (1, 1), (1, 1), 2)
    assert np.array_equal(cols[:, :2], base[:, :2])
    assert np.array_equal(cols[:, 2:, :, :, :-1], base[:, 2:, :, :, 1:])


# ----------------------------------------------------------------------------------------------------------------
# deformable PS-RoI pooling
# ----------------------------------------------------------------------------------------------------------------
def brute_pool(x, rois, trans, spatial_scale, output_dim, group_size, pooled, part_size, spp, trans_std, no_trans):
    """DeformablePSROIPoolForwardKernel (dcn_v2_psroi_pooling_cuda.cu:59-146) one output element at a time, every
    value an np.float32 scalar so that every operation rounds to fp32 like the reference's `float`."""
    N, C, H, W = x.shape
    R = rois.shape[0]
    ncls = 1 if no_trans else trans.shape[1] // 2
    each = output_dim // ncls
    out = np.zeros((R, output_dim, pooled, pooled), f32)
    cnt = np.zeros(out.shape, np.int64)

    def rnd(v):   # C round(): half away from zero
        return f32(np.sign(v) * np.floor(abs(float(v)) + 0.5))

    for n in range(R):
        roi = rois[n]
        b = int(roi[0])
        s = f32(spatial_scale)
        sw, sh = rnd(roi[1]) * s - f32(0.5), rnd(roi[2]) * s - f32(0.5)
        ew, eh = (rnd(roi[3]) + f32(1)) * s - f32(0.5), (rnd(roi[4]) + f32(1)) * s - f32(0.5)
        rw, rh = max(ew - sw, f32(0.1)), max(eh - sh, f32(0.1))
        bw, bh = rw / f32(pooled), rh / f32(pooled)
        subw, subh = bw / f32(spp), bh / f32(spp)
        for ctop in range(output_dim):
            for ph in range(pooled):
                for pw in range(pooled):
                    part_h = int(np.floor(f32(ph) / f32(pooled) * f32(part_size)))
                    part_w = int(np.floor(f32(pw) / f32(pooled) * f32(part_size)))
                    cls = ctop // each
                    tx = f32(0) if no_trans else trans[n, 2 * cls, part_h, part_w] * f32(trans_std)
                    ty = f32(0) if no_trans else trans[n, 2 * cls + 1, part_h, part_w] * f32(trans_std)
                    ws = f32(pw) * bw + sw
                    ws = ws + tx * rw
                    hs = f32(ph) * bh + sh
                    hs = hs + ty * rh
                    gw = min(max(int(np.floor(f32(pw) * f32(group_size) / f32(pooled))), 0), group_size - 1)
                    gh = min(max(int(np.floor(f32(ph) * f32(group_size) / f32(pooled))), 0), group_size - 1)
                    c = (ctop * group_size + gh) * group_size + gw
                    acc, k = f32(0), 0
                    for ih in range(spp):
                        for iw in range(spp):
                            w = ws + f32(iw) * subw
                            h = hs + f32(ih) * subh
                            if w < -0.5 or w > W - 0.5 or h < -0.5 or h > H - 0.5:
                                continue
                            w = f32(min(max(w, 0.0), W - 1.0))
                            h = f32(min(max(h, 0.0), H - 1.0))
                            x1, x2, y1, y2 = int(np.floor(w)), int(np.ceil(w)), int(np.floor(h)), int(np.ceil(h))
                            dx, dy = w - f32(x1), h - f32(y1)
                            img = x[b, c]
                            val = (f32(1) - dx) * (f32(1) - dy) * img[y1, x1] + (f32(1) - dx) * dy * img[y2, x1] \
                                + dx * (f32(1) - dy) * img[y1, x2] + dx * dy * img[y2, x2]
                            acc = acc + val
                            k += 1
                    out[n, ctop, ph, pw] = f32(0) if k == 0 else acc / f32(k)
                    cnt[n, ctop, ph, pw] = k
    return out, cnt


def pool_case(r, N=2, output_dim=4, group_size=1, H=12, W=10, R=6, ncls=1, part=3, scale=0.5):
    x = r.standard_normal((N, output_dim * group_size ** 2, H, W)).astype(f32)
    xy = r.uniform(-6, 2 * W + 4, size=(R, 2))
    wh = r.uniform(0, 14, size=(R, 2))
    rois = np.concatenate([r.randint(0, N, size=(R, 1)), xy, xy + wh], 1).astype(f32)
    trans = r.standard_normal((R, 2 * ncls, part, part)).astype(f32)
    return x, rois, trans


@pytest.mark.parametrize("no_trans,group_size,ncls,pooled,part,spp", [
    (True, 1, 1, 3, 3, 4), (False, 1, 2, 3, 3, 2), (False, 3, 2, 3, 2, 1), (False, 2, 4, 5, 3, 3)])
def test_pool_restatement_equals_scalar_brute_force(no_trans, group_size, ncls, pooled, part, spp):
    r = np.random.RandomState(pooled * 10 + group_size + ncls)
    x, rois, trans = pool_case(r, output_dim=4, group_size=group_size, ncls=ncls, part=part)
    args = (0.5, 4, group_size, pooled, part, spp, 0.3)
    got32, cnt32, _ = psroi_pool(x, rois, trans, *args, no_trans, acc=np.float32)
    want, cnt = brute_pool(x, rois, trans, *args, no_trans)
    assert np.array_equal(cnt32, cnt)
    # the geometry is the same to the bit; the blend's order of products may differ by an fp32 rounding or two
    assert np.allclose(got32, want, rtol=1e-5, atol=1e-6)
    got64, cnt64, mag = psroi_pool(x, rois, trans, *args, no_trans)
    assert np.array_equal(cnt64, cnt) and (cnt == 0).any() and (cnt == spp * spp).any()
    assert np.all(np.abs(got64 - want) <= 2.0 ** -20 * (spp * spp + 8) * mag + 1e-30)


def test_pool_hand_derived_cases():
    # constant input: every counted bin is the constant, every empty bin 0
    x = np.full((1, 2, 8, 8), 3.25, f32)
    rois = np.array([[0, 2, 2, 9, 9], [0, 40, 40, 50, 50], [0, -20, -20, 3, 3]], f32)
    out, cnt, _ = psroi_pool(x, rois, None, 0.5, 2, 1, 3, 3, 2, 0.0, True)
    assert np.all(out[cnt > 0] == 3.25) and np.all(out[cnt == 0] == 0)
    assert (cnt[1] == 0).all()                   # wholly outside the map
    assert (cnt[0] == 4).all()
    # one sample per bin is the bilinear value at the bin's start: a 1x1 bin of a 1-pixel RoI at (x, y) = (2, 3) of a
    # ramp, scale 1: start = 2 - 0.5 = 1.5 -> halfway between columns 1 and 2
    ramp = (np.arange(8)[None, :] * 10.0 + np.arange(8)[:, None]).astype(f32)[None, None]
    out, cnt, _ = psroi_pool(ramp, np.array([[0, 2, 3, 2, 3]], f32), None, 1.0, 1, 1, 1, 1, 1, 0.0, True)
    assert cnt[0, 0, 0, 0] == 1 and out[0, 0, 0, 0] == 0.5 * (ramp[0, 0, 2, 1] + ramp[0, 0, 2, 2]) * 0.5 + \
        0.5 * (ramp[0, 0, 3, 1] + ramp[0, 0, 3, 2]) * 0.5
    # a degenerate RoI (end before start) is 0.1 wide: all its samples fall within 0.1 of its start (4.5, 4.5), where
    # the ramp is 44 + 0.5 * 11
    out, cnt, _ = psroi_pool(ramp, np.array([[0, 5, 5, 1, 1]], f32), None, 1.0, 1, 1, 2, 2, 2, 0.0, True)
    assert (cnt == 4).all() and np.all(np.abs(out - (ramp[0, 0, 4, 4] + 0.5 * 11)) <= 0.1 * 11)


def test_pool_round_is_half_away_from_zero():
    """Corners at .5 round away from zero (C round()), not to even (numpy's round)."""
    x = np.arange(16 * 16, dtype=f32).reshape(1, 1, 16, 16)
    for v, want in ((2.5, 3), (3.5, 4), (-0.5, -1), (0.49999997, 0)):
        rois = np.array([[0, v, 4, v, 4]], f32)
        out, _, _ = psroi_pool(x, rois, None, 1.0, 1, 1, 1, 1, 1, 0.0, True)
        ref, _, _ = psroi_pool(x, np.array([[0, want, 4, want, 4]], f32), None, 1.0, 1, 1, 1, 1, 1, 0.0, True)
        assert out[0, 0, 0, 0] == ref[0, 0, 0, 0], v


def test_dcn_v2_module_exports_every_name_the_reference_script_imports(tmp_path, monkeypatch):
    """external/DCNv2/test.py:11-12 against a `dcn_v2` that is this package's module (a one-line shim on sys.path)."""
    import importlib
    import sys
    (tmp_path / "dcn_v2.py").write_text("from yolact_b200.dcn_v2 import *  # noqa: F401,F403\n"
                                        "from yolact_b200.dcn_v2 import dcn_v2_conv, dcn_v2_pooling  # noqa: F401\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    monkeypatch.delitem(sys.modules, "dcn_v2", raising=False)
    mod = importlib.import_module("dcn_v2")
    for name in ("dcn_v2_conv", "DCNv2", "DCN", "dcn_v2_pooling", "DCNv2Pooling", "DCNPooling"):
        assert callable(getattr(mod, name)), name
    p = mod.DCNPooling(1.0 / 4, 7, 32, False, trans_std=0.1, deform_fc_dim=64)
    assert [k for k, _ in p.named_parameters()] == ["offset_mask_fc.%d.%s" % (i, w) for i in (0, 2, 4)
                                                    for w in ("weight", "bias")]
