"""FastMaskIoUNet through yb_maskiou, against float64 (tests/resample_reference.py maskiou_f64), through both of its
entries: net.maskiou_net(x) (the per-channel map, FastMaskIoUNet.forward) and the per-row gather postprocess's
rescoring uses (output_utils._maskiou_rescore).

The maskiou_net weights are seeded mixed-sign ones (the network's deterministic weights elsewhere), checked to leave
20-80 % of every layer's pre-activations negative, so that each ReLU is exercised.  Every output is judged against
K * 2^-24 * M, M the magnitude chain (the same convs on |x| with |w| and |b|), never against the tensor's range.

Also: the gather equals the map's channel bit for bit; a row's result does not depend on the other rows of the call;
the f32 and f16x3 handles (both run the fp32 CUDA-core kernels) give identical bits; a 600x600 mask, whose last map
(17 x 17) spreads its maxima over all four warps of the final reduction; and masks under 63 pixels on either axis,
which nn.Conv2d refuses, are refused.
"""
import ctypes

import numpy as np
import pytest
import torch

import yolact_b200
from oracle.weights import deterministic_state_dict
from tests import resample_reference as R
from tests.error_bounds import U24, worst
from tests.helpers import cfg_for
from yolact_b200 import _lib
from yolact_b200.output_utils import _maskiou_rescore

pytestmark = pytest.mark.gpu

NC = 80            # num_classes - 1 output channels
# M is a worst case that every rounding error aligns with |w| through all six layers (M is about 1e5 times the outputs
# here); the fp32 accumulation errors are random-signed and stay far below one unit of it.  One unit keeps the bound
# under a third of the gaps between the final max's per-warp stripes (see the 600 x 600 test).
K_BOUND = 1.0
KEYS = ["maskiou_net.maskiou_net.%d" % i for i in (0, 2, 4, 6, 8, 10)]
RATIO = [0.0]


@pytest.fixture(scope="module", autouse=True)
def report_ratio():
    yield
    print("maskiou: largest err / (2^-24 * M): %.3g" % RATIO[0])


def seeded_weights():
    """He-scaled N(0, 1) weights and N(0, 0.1) biases for the six maskiou_net convs."""
    r = np.random.RandomState(11)
    shapes = [(8, 1, 3), (16, 8, 3), (32, 16, 3), (64, 32, 3), (128, 64, 3), (NC, 128, 1)]
    ws, bs = [], []
    for co, ci, k in shapes:
        ws.append((r.standard_normal((co, ci, k, k)) * (2.0 / (ci * k * k)) ** 0.5).astype(np.float32))
        bs.append((r.standard_normal(co) * 0.1).astype(np.float32))
    return ws, bs


@pytest.fixture(scope="module")
def nets():
    cfg = cfg_for("yolact_plus_resnet50_config")
    yolact_b200.cfg.replace(cfg.copy())
    ws, bs = seeded_weights()
    out = {}
    for prec in ("f32", "f16x3"):
        net = yolact_b200.Yolact(cfg, precision=prec)
        sd = deterministic_state_dict(net.state_dict(), 0)
        for key, w, b in zip(KEYS, ws, bs):
            sd[key + ".weight"] = torch.from_numpy(w)
            sd[key + ".bias"] = torch.from_numpy(b)
        net.load_state_dict(sd)
        net.eval()
        out[prec] = net
    return out


def masks(kind, n, H, W, seed):
    """[n, H, W] fp32: cropped sigmoid-like masks in [0, 1] (what postprocess feeds), binary masks, all zeros, or one
    hot pixel in a corner (the four corners in turn)."""
    r = np.random.RandomState(seed)
    m = np.zeros((n, H, W), np.float32)
    if kind == "zeros":
        return m
    if kind == "corners":
        for i in range(n):
            m[i, (0, H - 1)[i % 2], (0, W - 1)[(i // 2) % 2]] = 1
        return m
    for i in range(n):
        y0, x0 = r.randint(0, H // 2), r.randint(0, W // 2)
        y1, x1 = r.randint(y0 + H // 4, H + 1), r.randint(x0 + W // 4, W + 1)
        m[i, y0:y1, x0:x1] = 1 / (1 + np.exp(-r.standard_normal((y1 - y0, x1 - x0)) * 3))
    if kind == "binary":
        m = (m > 0.5).astype(np.float32)
    return m


def reference(x):
    ws, bs = seeded_weights()
    return R.maskiou_f64(x, ws, bs)


def net_map(net, x):
    out = net.maskiou_net(torch.from_numpy(x).cuda().unsqueeze(1))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def net_gather(net, x, cls):
    """_maskiou_rescore with unit scores: the gathered maskiou itself."""
    pm = torch.from_numpy(x).cuda()
    rescored, _ = _maskiou_rescore(net, net.cfg, pm, torch.from_numpy(np.asarray(cls, np.int64)).cuda(),
                                   torch.ones(x.shape[0], device="cuda"))
    torch.cuda.synchronize()
    return rescored.cpu().numpy()


def check(got, want, mag, what):
    assert got.shape == want.shape, (got.shape, want.shape)
    err = np.abs(got.astype(np.float64) - want)
    tol = K_BOUND * U24 * mag
    ratio = float((err / (U24 * mag)).max()) if np.isfinite(err).all() else np.inf
    RATIO[0] = max(RATIO[0], ratio)
    print("%s: max err / (2^-24 * M) = %.3g" % (what, ratio))
    assert (err <= tol).all(), (what, worst(err, tol))


def classes(n, seed):
    c = np.random.RandomState(seed).randint(0, NC, n)
    c[0] = 0
    c[-1] = NC - 1
    return c


SIZES = [(63, 63), (64, 64), (138, 138), (176, 176), (64, 138), (138, 64)]


@pytest.mark.parametrize("kind", ["sigmoid", "binary", "zeros", "corners"])
@pytest.mark.parametrize("H,W", SIZES, ids=str)
def test_maskiou_map_and_gather(nets, H, W, kind):
    n = 37
    x = masks(kind, n, H, W, H * W)
    want, mag, _ = reference(x)
    got = net_map(nets["f16x3"], x)
    check(got, want, mag, "maskiou %dx%d %s n=%d" % (H, W, kind, n))
    assert np.array_equal(net_map(nets["f32"], x).view(np.uint32), got.view(np.uint32)), "f32 and f16x3 handles differ"
    cls = classes(n, H + W)
    g = net_gather(nets["f16x3"], x, cls)
    assert np.array_equal(g.view(np.uint32), R.maskiou_gather(got, cls).view(np.uint32)), "gather != map channel"


def test_maskiou_weights_exercise_every_relu():
    x = masks("sigmoid", 37, 138, 138, 138 * 138)
    _, _, pre = reference(x)
    for i, z in enumerate(pre):
        frac = (z < 0).mean()
        assert 0.2 <= frac <= 0.8, (KEYS[i], frac)


@pytest.mark.parametrize("H,W", [(138, 138), (63, 64)], ids=str)
def test_maskiou_rows_are_independent_of_the_batch(nets, H, W):
    """Row i alone (n = 1) and within 300 rows gives the same bits, in both entries (display.py runs maskiou_net over
    padded rows at once and relies on this)."""
    n = 300
    x = masks("sigmoid", n, H, W, 5)
    cls = classes(n, 6)
    net = nets["f16x3"]
    full = net_map(net, x)
    full_g = net_gather(net, x, cls)
    want, mag, _ = reference(x)
    check(full, want, mag, "maskiou %dx%d n=300" % (H, W))
    for i in (0, 1, 150, 299):
        one = net_map(net, x[i:i + 1])
        assert np.array_equal(one.view(np.uint32), full[i:i + 1].view(np.uint32)), i
        one_g = net_gather(net, x[i:i + 1], cls[i:i + 1])
        assert np.array_equal(one_g.view(np.uint32), full_g[i:i + 1].view(np.uint32)), i


def test_maskiou_600_every_warp_of_the_final_max(nets):
    """600 x 600 -> a 17 x 17 last map: each of maxpool_gather's 4 warps reduces a stripe of pixels (pixel mod 128 in
    32-wide ranges).  The reference shows that for every warp some (row, channel) has its maximum in that warp's stripe
    only, above the other stripes by more than twice the tolerance."""
    n = 2
    x = masks("sigmoid", n, 600, 600, 600)
    x[:, 100:500, 100:500] = 1 / (1 + np.exp(-np.random.RandomState(7).standard_normal((n, 400, 400)) * 3))
    want, mag, pre = reference(x)
    last = np.maximum(pre[-1], 0).reshape(n, -1, NC)          # [n, 289, C]
    assert last.shape[1] == 289
    stripe = (np.arange(289) % 128) // 32
    smax = np.stack([last[:, stripe == w].max(axis=1) for w in range(4)])   # [4, n, C]
    tol = K_BOUND * U24 * mag
    for w in range(4):
        others = np.delete(smax, w, axis=0).max(axis=0)
        assert ((smax[w] - others) > 2 * tol).any(), "no maximum lies in warp %d's stripe alone" % w
    cls = np.array([5, 79])
    for net in nets.values():
        got = net_map(net, x)
        check(got, want, mag, "maskiou 600x600 n=2 %s" % net.precision_name)
        g = net_gather(net, x, cls)
        assert np.array_equal(g.view(np.uint32), R.maskiou_gather(got, cls).view(np.uint32))


def c_maskiou(net, x, cls=None):
    """yb_maskiou straight through the C ABI; x [n, ph, pw] fp32 on the device."""
    lib = _lib.load()
    n, ph, pw = x.shape
    out = torch.full((max(n, 1),) if cls is not None else (max(n, 1), NC), float("nan"), device="cuda")
    _lib.check(lib.yb_maskiou(net._handle_for(x.device), _lib.ptr(x), n, ph, pw, _lib.ptr(cls), _lib.ptr(out),
                              _lib.current_stream()), "yb_maskiou")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("axis", ["H", "W"])
def test_maskiou_refuses_masks_under_63_pixels(nets, axis):
    """nn.Conv2d refuses 47..62 (its fifth conv would get 1 or 2 rows); smaller sizes were refused already."""
    net = nets["f16x3"]
    cls = torch.zeros(2, dtype=torch.int64, device="cuda")
    for s in range(40, 64):
        shape = (2, s, 63) if axis == "H" else (2, 63, s)
        x = torch.rand(shape, device="cuda")
        if s >= R.MASKIOU_MIN_SIZE:
            assert torch.isfinite(c_maskiou(net, x, cls)).all()
            assert torch.isfinite(net.maskiou_net(x.unsqueeze(1))).all()
            continue
        with pytest.raises(_lib.YbError, match="mask too small"):
            c_maskiou(net, x, cls)
        with pytest.raises(_lib.YbError, match="mask too small"):
            c_maskiou(net, x)
        with pytest.raises(_lib.YbError, match="mask too small"):
            net.maskiou_net(x.unsqueeze(1))


def test_maskiou_no_rows(nets):
    net = nets["f16x3"]
    out = net.maskiou_net(torch.zeros(0, 1, 138, 138, device="cuda"))
    assert out.shape == (0, NC)
    x = torch.zeros(1, 138, 138, device="cuda")
    lib = _lib.load()
    before = lib.yb_launch_count(net._handle_for(x.device))
    _lib.check(lib.yb_maskiou(net._handle_for(x.device), _lib.ptr(x), 0, 138, 138, None, _lib.ptr(x),
                              _lib.current_stream()), "yb_maskiou")
    assert lib.yb_launch_count(net._handle_for(x.device)) == before
    assert (x == 0).all()
