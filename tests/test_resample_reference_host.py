"""The float64 references of tests/resample_reference.py against torch's own CPU operators (no GPU needed): the max
pool bit for bit, the bilinear resample at every ratio the network runs, FastMaskIoUNet as the reference's nn.Sequential
builds it, the mask sizes nn.Conv2d refuses, and the split-precision encoder."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import resample_reference as R

# (H, W) -> (Ho, Wo): the FPN's top-down resizes (550, 700, 160 and 256x320 inputs), the protonet's x2 and edge shapes
FPN_RESIZES = [((18, 18), (35, 35)), ((35, 35), (69, 69)), ((22, 22), (44, 44)), ((44, 44), (88, 88)),
               ((5, 5), (10, 10)), ((10, 10), (20, 20)), ((8, 10), (16, 20)), ((16, 20), (32, 40))]
PROTO_RESIZES = [((69, 69), (138, 138)), ((88, 88), (176, 176)), ((35, 35), (70, 70))]
EDGE_RESIZES = [((1, 1), (2, 2)), ((1, 7), (3, 13)), ((9, 5), (17, 11)), ((12, 12), (12, 12))]


def nchw(x):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x).transpose(0, 3, 1, 2)))


@pytest.mark.parametrize("H,W", [(1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (16, 20), (35, 34)], ids=str)
def test_maxpool_reference_is_torch_max_pool2d_bit_for_bit(H, W):
    r = np.random.RandomState(H * 100 + W)
    x = (r.standard_normal((2, H, W, 8)) * 3).astype(np.float32)
    x[1] = -np.abs(x[1]) - 1         # every window all-negative, the border ones included
    want = F.max_pool2d(nchw(x), 3, 2, 1).permute(0, 2, 3, 1).numpy()
    got = R.maxpool3x3s2_f64(x).astype(np.float32)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("src,dst", FPN_RESIZES + PROTO_RESIZES + EDGE_RESIZES, ids=str)
def test_bilinear_reference_agrees_with_interpolate(src, dst):
    r = np.random.RandomState(src[0] * 1000 + dst[1])
    x = r.standard_normal((2, src[0], src[1], 4)).astype(np.float32)
    want = F.interpolate(nchw(x), size=dst, mode="bilinear", align_corners=False).permute(0, 2, 3, 1).numpy()
    got, scale = R.bilinear_f64(x, *dst)
    err = np.abs(got - want.astype(np.float64))
    # ATen's CPU build may contract scale * (o + 0.5) - 0.5 into an FMA, which the kernel (and the reference) do not:
    # the source coordinate s, and with it each lambda, may then differ by an ulp of s
    geometry = 2 * 2.0 ** -24 * (max(src) + 1) * np.abs(x).max()
    assert (err <= 4 * 2.0 ** -24 * scale + geometry).all(), float((err / scale).max())


def test_bilinear_reference_x2_is_interpolate_scale_factor_2():
    """The protonet's InterpolateModule(scale_factor=2): ATen's scale is 1 / 2, the same fp32 value as in / (2 in)."""
    x = np.random.RandomState(3).standard_normal((1, 35, 35, 4)).astype(np.float32)
    want = F.interpolate(nchw(x), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1).numpy()
    got, scale = R.bilinear_f64(x, 70, 70)
    assert (np.abs(got - want) <= 4 * 2.0 ** -24 * scale).all()


def test_bilinear_taps_at_the_last_row():
    """Upsampling, the last outputs read the last source row twice (i1 stays at n_in - 1) with l1 > 0; the identity
    resize reads each row once with l1 = 0."""
    i0, i1, l0, l1 = R.bilinear_taps(18, 35)
    assert i0[-1] == 17 and i1[-1] == 17 and l1[-1] > 0
    assert (i1 <= 17).all() and (l0 + l1 == 1).all()
    i0, i1, l0, l1 = R.bilinear_taps(12, 12)
    assert (i0 == np.arange(12)).all() and (l1 == 0).all()


def reference_maskiou_net(num_classes=81):
    """maskiou_net as the reference's make_net builds it: [Conv2d(., ., 3, stride=2), ReLU] x 5, Conv2d(128, C-1, 1),
    ReLU, in float64 with seeded mixed-sign weights."""
    chans = [1, 8, 16, 32, 64, 128]
    layers = []
    for i in range(5):
        layers += [nn.Conv2d(chans[i], chans[i + 1], 3, stride=2), nn.ReLU(inplace=True)]
    layers += [nn.Conv2d(128, num_classes - 1, 1), nn.ReLU(inplace=True)]
    net = nn.Sequential(*layers).double()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for m in net:
            if isinstance(m, nn.Conv2d):
                fan_in = m.weight[0].numel()
                m.weight.copy_(torch.randn(m.weight.shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g, dtype=torch.float64) * 0.1)
    return net


@pytest.mark.parametrize("H,W", [(63, 63), (64, 138), (70, 65)], ids=str)
def test_maskiou_reference_is_the_reference_network(H, W):
    net = reference_maskiou_net()
    convs = [m for m in net if isinstance(m, nn.Conv2d)]
    masks = np.random.RandomState(H + W).uniform(0, 1, (3, H, W))
    cls = np.array([0, 79, 41])
    with torch.no_grad():
        x = net(torch.from_numpy(masks).unsqueeze(1))
        want = F.max_pool2d(x, x.size()[2:]).squeeze(-1).squeeze(-1)
        want_g = torch.gather(want, 1, torch.from_numpy(cls).view(-1, 1)).view(-1)
    out, mag, pre = R.maskiou_f64(masks, [c.weight.detach().numpy() for c in convs], [c.bias.detach().numpy() for c in convs])
    np.testing.assert_allclose(out, want.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(R.maskiou_gather(out, cls), want_g.numpy(), rtol=1e-12, atol=1e-12)
    assert (mag >= np.abs(out)).all()
    assert [p.shape[1] for p in pre] == R.maskiou_out_size(H)


def c_truncating_out(n, k, s):
    """(n - k) / s + 1 as C evaluates it (division truncating toward zero)."""
    return int((n - k) / s) + 1


def test_maskiou_minimum_mask_size_is_63():
    """nn.Conv2d refuses mask sides 47..62 (the fifth conv would see 1 or 2 rows), accepts 63.  C's truncating
    (n - 3) / 2 + 1 gives 1 for n = 2 and so accepts exactly those sizes: the range the library must refuse itself."""
    net = reference_maskiou_net()
    for n in range(40, 64):
        c_accepts = True
        m = n
        for k, s in R.MASKIOU_LAYERS:
            m = c_truncating_out(m, k, s)
            c_accepts &= m >= 1
        for shape in ((n, 63), (63, n)):
            x = torch.zeros((1, 1) + shape, dtype=torch.float64)
            if n >= R.MASKIOU_MIN_SIZE:
                assert net(x).shape[2:] == (1, 1)
                assert R.maskiou_out_size(n) is not None
            else:
                with pytest.raises(RuntimeError):
                    net(x)
                assert R.maskiou_out_size(n) is None
        assert c_accepts == (n >= 47), n


def test_split_encoder_round_trips_within_2_pow_minus_22():
    r = np.random.RandomState(0)
    v = (np.exp2(r.uniform(-14, np.log2(65504), 200000)) * r.choice([-1, 1], 200000)).astype(np.float32)
    v = np.concatenate([v, np.float32([65504, -65504, 2.0 ** -14, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11])])
    hi, lo = R.split_encode(v)
    assert hi.dtype == lo.dtype == np.float16
    back = R.split_decode(hi, lo).astype(np.float64)
    assert (np.abs(back - v) <= 2.0 ** -22 * np.abs(v)).all()
    assert (hi.astype(np.float32) == v.astype(np.float16).astype(np.float32)).all()   # hi is fp16 round-to-nearest-even
    assert hi[-2] == 1 and hi[-1] == np.float16(1 + 2.0 ** -9)   # the two ties go to the even neighbour


def test_encoders_saturate_at_65504():
    v = np.float32([65505, 70000, 1e30, np.inf, -70000, -np.inf])
    hi, lo = R.split_encode(v)
    assert (hi == np.float16([65504] * 4 + [-65504] * 2)).all() and (lo == 0).all()
    assert (R.f16_encode(v) == hi).all()
    raw = R.encode_nhwc(np.float32([[[[3.0, -70000.0]]]]), "f16x3")
    assert raw.shape == (1, 1, 1, 4) and (R.decode_nhwc(raw, "f16x3") == [[[[3.0, -65504.0]]]]).all()
