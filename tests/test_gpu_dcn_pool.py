"""Deformable PS-RoI pooling on the GPU (yb_dcn_psroi_pool, dcn_v2_pooling / DCNv2Pooling / DCNPooling) judged per
element against the float64 restatement tests/dcn_general_reference.psroi_pool (the reference kernel's fp32 geometry;
checked on the CPU against a scalar brute force): the sample counts exactly, the values within a few fp32 roundings of
the magnitude they average, |y - ref| <= (8 + 2 * spp^2) * 2^-24 * mag."""
import ctypes

import numpy as np
import pytest
import torch

from tests.dcn_general_reference import psroi_pool
from tests.error_bounds import worst
from yolact_b200 import _lib
from yolact_b200.dcn_v2 import DCNPooling, DCNv2Pooling, _handle, dcn_v2_pooling

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1
SENTINEL = -12345.0
f32 = np.float32


def pool_abi(x, rois, trans, out, count, N, C, H, W, R, no_trans, ncls, scale, output_dim, group_size, pooled, part,
             spp, trans_std, null=()):
    ptr = lambda name, a: ctypes.c_void_p(0) if (name in null or a is None) else _lib.ptr(a)
    return _lib.load().yb_dcn_psroi_pool(_handle(out.device, _lib.YB_PREC_F32), ptr("input", x), ptr("rois", rois),
                                         ptr("trans", trans), ptr("output", out), ptr("count", count), N, C, H, W, R,
                                         no_trans, ncls, scale, output_dim, group_size, pooled, part, spp, trans_std,
                                         _lib.current_stream(out.device))


def run_and_check(x, rois, trans, scale, output_dim, group_size, pooled, part, spp, trans_std, no_trans, what=""):
    N, C, H, W = x.shape
    R = rois.shape[0]
    ncls = 1 if no_trans else trans.shape[1] // 2
    out = torch.full((R, output_dim, pooled, pooled), SENTINEL, device="cuda")
    cnt = torch.full_like(out, SENTINEL)
    tt = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    xd, rd, td = tt(x), tt(rois), tt(None if no_trans else trans)
    st = pool_abi(xd, rd, td, out, cnt, N, C, H, W, R, int(no_trans), ncls, scale, output_dim, group_size, pooled,
                  part, spp, trans_std)
    assert st == 0, _lib.load().yb_last_error()
    ref, ref_cnt, mag = psroi_pool(x, rois, trans, scale, output_dim, group_size, pooled, part, spp, trans_std,
                                   no_trans)
    y, c = out.cpu().numpy(), cnt.cpu().numpy()
    assert np.array_equal(c, ref_cnt.astype(f32)), what
    err = np.abs(y - ref)
    tol = (8 + 2 * spp * spp) * 2.0 ** -24 * mag + 1e-37
    assert (err <= tol).all(), (what, worst(err, tol))
    assert (y[ref_cnt == 0] == 0).all()
    # the module-level function computes the same bits
    y2 = dcn_v2_pooling(xd, rd, td if td is not None else xd.new(), scale, pooled, output_dim, no_trans, group_size,
                        part, spp, trans_std)
    assert torch.equal(y2, out)
    return y, ref_cnt


def pool_case(r, N, output_dim, group_size, H, W, R, ncls, part):
    x = r.standard_normal((N, output_dim * group_size ** 2, H, W)).astype(f32)
    xy = r.uniform(-20, 2 * max(H, W) + 10, size=(R, 2))
    wh = r.uniform(0, 40, size=(R, 2))
    rois = np.concatenate([r.randint(0, N, size=(R, 1)), xy, xy + wh], 1).astype(f32)
    trans = r.standard_normal((R, 2 * ncls, part, part)).astype(f32)
    return x, rois, trans


@pytest.mark.parametrize("no_trans,group_size,ncls,pooled,part,spp", [
    (True, 1, 1, 7, 7, 4), (True, 3, 1, 3, 3, 1), (False, 1, 1, 7, 7, 4), (False, 1, 4, 7, 7, 1),
    (False, 3, 2, 6, 4, 4), (False, 3, 4, 3, 5, 2), (False, 1, 2, 5, 3, 4)])
def test_pooling_vs_float64(no_trans, group_size, ncls, pooled, part, spp):
    r = np.random.RandomState(100 * pooled + 10 * group_size + ncls + part)
    x, rois, trans = pool_case(r, 3, 8, group_size, 17, 23, 40, ncls, part)
    _, cnt = run_and_check(x, rois, trans, 0.5, 8, group_size, pooled, part, spp, 0.2, no_trans)
    assert (cnt == 0).any() and (cnt == spp * spp).any() and len(np.unique(rois[:, 0])) == 3


def test_roi_edges_degenerate_and_half_corners():
    """RoIs partly and wholly outside the map, degenerate ones (end before start: size clamped to 0.1) and corners at
    .5 (round() half away from zero) on both sides of zero."""
    r = np.random.RandomState(3)
    N, H, W = 2, 16, 12
    x = r.standard_normal((N, 4, H, W)).astype(f32)
    rois = np.array([
        [0, -10, -10, 12, 12], [1, 20, 25, 60, 70], [0, 100, 100, 120, 120], [1, -50, -10, -20, 30],
        [0, 8, 8, 2, 2], [1, 4, 4, 4, 4], [0, 7, 7, 7.4, 3],
        [0, 2.5, 3.5, 10.5, 11.5], [1, -0.5, -1.5, 0.5, 1.5], [0, 6.49999, 6.5, 13.5, 14.50001],
    ], f32)
    trans = r.standard_normal((len(rois), 2, 3, 3)).astype(f32)
    for no_trans in (True, False):
        _, cnt = run_and_check(x, rois, trans, 0.5, 4, 1, 3, 3, 4, 0.1, no_trans, "edges")
        assert (cnt[2] == 0).all() and (cnt[3] == 0).all()      # wholly outside
        assert (cnt[0] > 0).any() and (cnt[0] < 16).any()      # partly outside


# ----------------------------------------------------------------------------------------------------------------
# the reference script's pooling checks and examples (external/DCNv2/test.py:100-131, 183-250)
# ----------------------------------------------------------------------------------------------------------------
def test_check_pooling_zero_offset():
    x = torch.zeros(2, 16, 64, 64)
    x[0, :, 16:26, 16:26] = 1.
    x[1, :, 10:20, 20:30] = 2.
    rois = torch.tensor([[0, 65, 65, 103, 103], [1, 81, 41, 119, 79]]).float()
    xd, rd = x.cuda(), rois.cuda()
    pooling = DCNv2Pooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=16, no_trans=True, group_size=1,
                           trans_std=0.0).cuda()
    out = pooling(xd, rd, xd.new())
    dpooling = DCNv2Pooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=16, no_trans=False, group_size=1,
                            trans_std=0.0).cuda()
    dout = dpooling(xd, rd, torch.zeros(20, 2, 7, 7).cuda()[:2])
    ref, _, _ = psroi_pool(x.numpy(), rois.numpy(), None, 0.25, 16, 1, 7, 7, 4, 0.0, True)
    assert out.shape == dout.shape == (2, 16, 7, 7)
    assert np.allclose(out.cpu().numpy(), ref, rtol=1e-6, atol=1e-7)
    assert torch.equal(out, dout)               # trans_std 0: the offsets change nothing
    # the means the script prints: the RoIs cover the squares exactly (1.0 and 2.0 where they lie)
    assert out[0].mean().item() > 0 and out[1].mean().item() > 0


def example_inputs(seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 32, 64, 64, generator=g)
    batch_inds = torch.randint(2, (20, 1), generator=g).float()
    xx = torch.randint(256, (20, 1), generator=g).float()
    yy = torch.randint(256, (20, 1), generator=g).float()
    w = torch.randint(64, (20, 1), generator=g).float()
    h = torch.randint(64, (20, 1), generator=g).float()
    rois = torch.cat((batch_inds, xx, yy, xx + w, yy + h), dim=1)
    return x, rois, torch.randn(20, 2, 7, 7, generator=g)


def test_example_dpooling():
    x, rois, offset = example_inputs(1)
    pooling = DCNv2Pooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=32, no_trans=True, group_size=1,
                           trans_std=0.1).cuda()
    dpooling = DCNv2Pooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=32, no_trans=False, group_size=1,
                            trans_std=0.1).cuda()
    out = pooling(x.cuda(), rois.cuda(), offset.cuda())
    dout = dpooling(x.cuda(), rois.cuda(), offset.cuda())
    assert out.shape == dout.shape == (20, 32, 7, 7)
    for y, no_trans in ((out, True), (dout, False)):
        ref, _, mag = psroi_pool(x.numpy(), rois.numpy(), offset.numpy(), 0.25, 32, 1, 7, 7, 4, 0.1, no_trans)
        err = np.abs(y.cpu().numpy() - ref)
        assert (err <= 40 * 2.0 ** -24 * mag + 1e-37).all()
    assert not torch.equal(out, dout)


def test_example_mdpooling():
    """DCNPooling(no_trans=False): plain pooling -> offset_mask_fc -> deformable pooling * sigmoid(mask), with the
    MLP's weights seeded (its last layer starts at zero, which would make the offsets zero)."""
    x, rois, _ = example_inputs(2)
    torch.manual_seed(5)
    dp = DCNPooling(spatial_scale=1.0 / 4, pooled_size=7, output_dim=32, no_trans=False, group_size=1, trans_std=0.1,
                    deform_fc_dim=1024).cuda()
    assert [k for k, _ in dp.named_parameters()] == ["offset_mask_fc.%d.%s" % (i, p) for i in (0, 2, 4)
                                                     for p in ("weight", "bias")]
    with torch.no_grad():
        dp.offset_mask_fc[4].weight.normal_(0, 0.02)
        dp.offset_mask_fc[4].bias.normal_(0, 1.0)
        xd, rd = x.cuda(), rois.cuda()
        dout = dp(xd, rd)
        roi = dcn_v2_pooling(xd, rd, xd.new(), 0.25, 7, 32, True, 1, 7, 4, 0.1)
        om = dp.offset_mask_fc(roi.view(20, -1)).view(20, 3, 7, 7)
    assert dout.shape == (20, 32, 7, 7)
    ref_roi, _, _ = psroi_pool(x.numpy(), rois.numpy(), None, 0.25, 32, 1, 7, 7, 4, 0.1, True)
    assert np.allclose(roi.cpu().numpy(), ref_roi, rtol=1e-5, atol=1e-6)
    offset = torch.cat((om[:, 0:1], om[:, 1:2]), dim=1).cpu().numpy()
    assert np.abs(offset).max() > 0.1
    mask = torch.sigmoid(om[:, 2:3]).cpu().numpy()
    ref, _, mag = psroi_pool(x.numpy(), rois.numpy(), offset, 0.25, 32, 1, 7, 7, 4, 0.1, False)
    err = np.abs(dout.cpu().numpy() - ref * mask)
    assert (err <= 48 * 2.0 ** -24 * mag * mask + 1e-37).all()


# ----------------------------------------------------------------------------------------------------------------
# refusals
# ----------------------------------------------------------------------------------------------------------------
REFUSALS = [  # name, overrides, message
    ("batch-neg", {"b0": -1.0}, "batch index of RoI 0"),
    ("batch-N", {"b0": 2.0}, "batch index of RoI 0"),
    ("batch-nan", {"b0": float("nan")}, "batch index of RoI 0"),
    ("batch-inf", {"b0": float("inf")}, "batch index of RoI 0"),
    ("C", {"C": 6}, "C must be output_dim * group_size^2"),
    ("classes", {"ncls": 3}, "num_classes must be >= 1 and divide output_dim"),
    ("classes-0", {"ncls": 0}, "num_classes must be >= 1 and divide output_dim"),
    ("pooled-0", {"pooled": 0}, "pooled, group_size, part_size and sample_per_part must be >= 1"),
    ("part-0", {"part": 0}, "pooled, group_size, part_size and sample_per_part must be >= 1"),
    ("spp-0", {"spp": 0}, "pooled, group_size, part_size and sample_per_part must be >= 1"),
    ("null-input", {"null": ("input",)}, "null argument"),
    ("null-rois", {"null": ("rois",)}, "null argument"),
    ("null-trans", {"null": ("trans",)}, "null argument"),
    ("null-output", {"null": ("output",)}, "null argument"),
]


@pytest.mark.parametrize("name,over,message", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_return_invalid_and_leave_the_output(name, over, message):
    r = np.random.RandomState(0)
    N, C, H, W, R = 2, 4, 8, 8, 3
    x = torch.from_numpy(r.standard_normal((N, C, H, W)).astype(f32)).cuda()
    rois = torch.tensor([[1, 1, 1, 9, 9], [0, 2, 2, 5, 5], [1, 0, 0, 15, 15]], dtype=torch.float32)
    if "b0" in over:
        rois[0, 0] = over["b0"]
    rois = rois.cuda()
    trans = torch.zeros(R, 4, 3, 3, device="cuda")
    out = torch.full((R, 4, 3, 3), SENTINEL, device="cuda")
    cnt = torch.full_like(out, SENTINEL)
    st = pool_abi(x, rois, trans, out, cnt, N, over.get("C", C), H, W, R, 0, over.get("ncls", 2), 0.5, 4, 1,
                  over.get("pooled", 3), over.get("part", 3), over.get("spp", 2), 0.1, null=over.get("null", ()))
    assert st == YB_ERR_INVALID
    assert message in _lib.load().yb_last_error().decode()
    torch.cuda.synchronize()
    assert (out == SENTINEL).all() and (cnt == SENTINEL).all()
    rois[0, 0] = 0
    st = pool_abi(x, rois, trans, out, cnt, N, C, H, W, R, 0, 2, 0.5, 4, 1, 3, 3, 2, 0.1)
    assert st == 0 and torch.isfinite(out).all()
