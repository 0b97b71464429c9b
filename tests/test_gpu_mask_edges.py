"""Mask assembly (yb_postprocess, yb_postprocess_batch, yb_postprocess_list) pixel by pixel against the float64 reference
of tests/mask_reference.py, at the crop, value, resize, band and layout edges.

Every case is judged the same way, in all three mask formats:
  - every decided pixel equals the reference's v > 0.5, and at most 1e-5 of the pixels (plus 2) are undecided;
  - the outputs are poisoned before the call (fp32 NaN, u8 0xAB, bit words 0xFFFFFFFF) and sit between guard bands:
    afterwards every pixel is 0 or 1, the bits above out_w in each row's last word are 0, and the guards are untouched;
  - proto_masks is within the per-source bound inside the crop window and exactly +0.0 outside it;
  - boxes_px equals .long() of the reference's sanitize_coordinates, computed by torch on the same GPU."""
import ctypes

import numpy as np
import pytest
import torch

from tests import mask_reference as R
from yolact_b200 import _lib
from yolact_b200.output_utils import _ops_handle

pytestmark = pytest.mark.gpu

f32 = np.float32
FORMATS = ("f32", "u8", "bits")
FMT = {"f32": _lib.YB_MASK_F32, "u8": _lib.YB_MASK_U8, "bits": _lib.YB_MASK_BITS}
DTYPE = {"f32": torch.float32, "u8": torch.uint8, "bits": torch.int32}
POISON = {"f32": float("nan"), "u8": 0xAB, "bits": -1}
GUARD = 64                      # guard elements on each side: 256, 64 and 256 bytes, so the masks stay 16-byte aligned
WORST = {"pm_ratio": 0.0, "undecided": 0, "pixels": 0, "cases": 0}


def row_elems(fmt, w):
    return (w + 31) // 32 if fmt == "bits" else w


def poisoned(fmt, count):
    return torch.full((count,), POISON[fmt], dtype=DTYPE[fmt], device="cuda")


def bit_pattern(t):
    """Tensor contents as integers, so NaN poison compares equal to itself."""
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_guard(buf, fmt, lo, hi, what):
    seg = bit_pattern(buf[lo:hi])
    want = bit_pattern(poisoned(fmt, 1))
    assert bool((seg == want).all()), "%s: guard elements [%d, %d) written" % (what, lo, hi)


def to_pixels(masks, fmt, h, w, what):
    """Kernel masks [n, h, w] (or [n, h, words]) -> uint8 [n, h, w] numpy, asserting every pixel is 0 or 1 and the
    padding bits of the bit format are 0."""
    a = masks.cpu().numpy()
    if fmt == "bits":
        words = a.view(np.uint32)
        bits = ((words[..., None] >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8)
        bits = bits.reshape(a.shape[0], h, -1)
        assert not bits[:, :, w:].any(), "%s: padding bits above out_w set" % what
        return bits[:, :, :w]
    ok = (a == 0) | (a == 1)
    assert ok.all(), "%s: %d pixels neither 0 nor 1, e.g. %r" % (what, (~ok).sum(), a[~ok][:4])
    return a.astype(np.uint8)


def judge(got, v, e, what):
    dec, want = R.decide(v, e)
    und = int((~dec).sum())
    WORST["undecided"] += und
    WORST["pixels"] += v.size
    assert und <= 1e-5 * v.size + 2, "%s: %d of %d pixels undecided" % (what, und, v.size)
    bad = dec & (got.astype(bool) != want)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError("%s: %d decided pixels differ; first at %s: got %d, v %.9g, e %.3g" %
                             (what, bad.sum(), at, got[at], v[at], e[at]))


def torch_boxes_px(box, h, w):
    """output_utils.py:97-99: sanitize_coordinates(cast=False) at the output size, then .long(), by torch on the GPU."""
    b = torch.from_numpy(np.ascontiguousarray(box, f32)).cuda()

    def sanitize(a, c, size):
        a, c = a * size, c * size
        return torch.clamp(torch.min(a, c), min=0), torch.clamp(torch.max(a, c), max=size)

    x1, x2 = sanitize(b[:, 0], b[:, 2], w)
    y1, y2 = sanitize(b[:, 1], b[:, 3], h)
    return torch.stack([x1, y1, x2, y2], 1).long()


def judge_proto_masks(pm, proto, coef, box, crop, what):
    val, bound, keep = R.proto_reference(proto, coef, box, crop)
    got = pm.cpu().numpy()
    out = got[~keep]
    assert (out == 0).all() and not np.signbit(out).any(), "%s: proto_masks not +0.0 outside the window" % what
    err = np.abs(got.astype(np.float64) - val)
    assert (err[keep] <= bound[keep]).all(), "%s: proto_masks outside the bound, worst ratio %.3g" % (
        what, (err[keep] / bound[keep]).max())
    if keep.any():
        WORST["pm_ratio"] = max(WORST["pm_ratio"], float((err[keep] / bound[keep]).max()))


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check(proto, coef, box, h, w, crop=True, formats=FORMATS):
    """yb_postprocess of one image into poisoned outputs between guard bands, judged against the reference."""
    proto, coef, box = np.asarray(proto, f32), np.asarray(coef, f32), np.asarray(box, f32)
    ph, pw, k = proto.shape
    n = coef.shape[0]
    v, e = R.mask_reference(proto, coef, box, h, w, crop)
    want_px = torch_boxes_px(box, h, w)
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    tp, tc, tb = cuda(proto), cuda(coef), cuda(box)
    WORST["cases"] += 1
    for fmt in formats:
        what = "%dx%d<-%dx%dx%d n=%d crop=%d %s" % (h, w, ph, pw, k, n, crop, fmt)
        plane = h * row_elems(fmt, w)
        buf = poisoned(fmt, GUARD + n * plane + GUARD)
        boxes_px = torch.full((n, 4), -0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=dev)
        pm = torch.full((n, ph, pw), float("nan"), device=dev)
        _lib.check(lib.yb_postprocess(_ops_handle(dev, k), _lib.ptr(tp), ph, pw, k, _lib.ptr(tc), _lib.ptr(tb), n, h, w,
                                      int(crop), FMT[fmt], ctypes.c_void_p(buf[GUARD:].data_ptr()),
                                      _lib.ptr(boxes_px), _lib.ptr(pm), _lib.current_stream(dev)), what)
        torch.cuda.synchronize()
        assert_guard(buf, fmt, 0, GUARD, what)
        assert_guard(buf, fmt, GUARD + n * plane, buf.numel(), what)
        judge(to_pixels(buf[GUARD:GUARD + n * plane].view(n, h, -1), fmt, h, w, what), v, e, what)
        assert torch.equal(boxes_px, want_px), (what, boxes_px, want_px)
        judge_proto_masks(pm, proto, coef, box, crop, what)
    return v, e


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nmask edges: %d cases, %d of %d pixels undecided, largest proto_masks error/bound %.3f" %
          (WORST["cases"], WORST["undecided"], WORST["pixels"], WORST["pm_ratio"]))


# ---- inputs ------------------------------------------------------------------------------------------------------------
def random_case(seed, n, ph, pw, k, wh_max=0.8):
    r = np.random.RandomState(seed)
    proto = np.maximum(r.standard_normal((ph, pw, k)), 0).astype(f32)
    coef = np.tanh(r.standard_normal((n, k))).astype(f32)
    c, wh = r.uniform(0.0, 1.0, (n, 2)), r.uniform(0.02, wh_max, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(f32)
    return proto, coef, box


def saturated(seed, n, ph, pw, k=32):
    """Prototypes +2 and positive coefficients: the sigmoid is ~1 inside the window, so a mask edge is the crop edge
    and the lambdas decide it."""
    r = np.random.RandomState(seed)
    proto = (np.maximum(r.standard_normal((ph, pw, k)), 0) + 2).astype(f32)
    coef = (np.abs(np.tanh(r.standard_normal((n, k)))) + 0.5).astype(f32)
    return proto, coef


def edge_coords(size):
    """Relative coordinates whose product with size is an integer, and the floats one ulp either side of them."""
    out = []
    for j in (0, 1, size // 3, size // 2, size - 1, size):
        x = f32(j) / f32(size)
        out += [x, np.nextafter(x, f32(-1)), np.nextafter(x, f32(2))]
    return np.array(out, f32)


def geometry_boxes(ph, pw):
    xs, ys = edge_coords(pw), edge_coords(ph)
    r = np.random.RandomState(ph * 1000 + pw)
    boxes = []
    for i, x in enumerate(xs):   # every edge candidate as x1 and as x2, and the same for y
        y = ys[i % len(ys)]
        boxes.append([x, y, f32(0.8), f32(0.9)])
        boxes.append([f32(0.1), f32(0.05), x, y])
    cell = 1.0 / pw
    boxes += [
        [0, 0, 1, 1], [-0.3, -0.2, 1.4, 1.7], [-0.5, -0.5, 0, 0], [1, 1, 1.2, 1.3],       # full, beyond, at 0 and 1
        [0.5, 0.5, 0.5, 0.5], [0.25, 0.4, 0.25, 0.7],                                   # zero width: 2 cells of padding
        [0.6, 0.7, 0.2, 0.3], [0.9, 0.1, 0.3, 0.6],                                     # x1 > x2, y1 > y2
        [0.4, 0.4, 0.4 + 0.3 * cell, 0.4 + 0.6 / ph], [0.33, 0.5, 0.33 + 0.9 * cell, 0.52],   # under one cell
    ]
    for _ in range(6):
        c = r.uniform(-0.1, 1.1, 2)
        wh = r.uniform(0.0, 0.5, 2)
        boxes.append([c[0] - wh[0], c[1] - wh[1], c[0] + wh[0], c[1] + wh[1]])
    return np.array(boxes, f32)


# ---- crop geometry -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ph,pw,h,w", [(36, 52, 148, 204), (138, 138, 550, 550), (36, 52, 28, 44), (48, 40, 144, 136)])
@pytest.mark.parametrize("crop", [True, False])
def test_crop_geometry(ph, pw, h, w, crop):
    box = geometry_boxes(ph, pw)
    proto, coef = saturated(ph + pw + h, len(box), ph, pw)
    v, _ = check(proto, coef, box, h, w, crop)
    if crop:
        assert not (v > 0.5).all(axis=(1, 2)).all() and (v > 0.5).any()


# ---- value edges -------------------------------------------------------------------------------------------------------
def ramp_case(seed, n, ph, pw, k):
    """A lincomb that is an affine function of the position: each detection's 0.5 line crosses its window."""
    r = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.arange(ph, dtype=f32), np.arange(pw, dtype=f32), indexing="ij")
    proto = np.zeros((ph, pw, k), f32)
    proto[..., 0] = xx / pw * 8
    proto[..., 1] = yy / ph * 8
    proto[..., 2] = 1
    if k > 4:
        proto[..., 3:] = r.standard_normal((ph, pw, k - 3)) * 0.05
    coef = np.zeros((n, k), f32)
    coef[:, :2] = r.uniform(-1.5, 1.5, (n, 2))
    c, wh = r.uniform(0.2, 0.8, (n, 2)), r.uniform(0.2, 0.7, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(f32)
    # the zero of the lincomb at the box centre
    coef[:, 2] = -(coef[:, 0] * c[:, 0] * 8 + coef[:, 1] * c[:, 1] * 8)
    if k > 4:
        coef[:, 3:] = r.standard_normal((n, k - 3)) * 0.1
    return proto, coef.astype(f32), box


def checker_case(n, ph, pw, k):
    """+-8 per prototype cell: a swapped i0 / i1 or a wrong first prototype row flips pixels."""
    yy, xx = np.meshgrid(np.arange(ph), np.arange(pw), indexing="ij")
    proto = np.zeros((ph, pw, k), f32)
    proto[..., 0] = np.where((yy + xx) % 2 == 0, 8, -8)
    proto[..., 1] = np.where(yy % 3 == 0, 8, -8)
    coef = np.zeros((n, k), f32)
    coef[:, 0] = 1
    coef[1::2, 0], coef[1::2, 1] = 0, 1
    r = np.random.RandomState(n * 31 + ph)
    c, wh = r.uniform(0.2, 0.8, (n, 2)), r.uniform(0.1, 0.9, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(f32)
    box[0] = [0, 0, 1, 1]
    return proto, coef, box


@pytest.mark.parametrize("ph,pw,h,w,k", [(138, 138, 550, 550, 32), (48, 40, 203, 277, 4), (36, 52, 64, 96, 128),
                                         (138, 138, 101, 83, 4)])
def test_ramp_crossings(ph, pw, h, w, k):
    proto, coef, box = ramp_case(h + w, 10, ph, pw, k)
    v, _ = check(proto, coef, box, h, w)
    assert 0.05 < (v > 0.5).mean() < 0.5


@pytest.mark.parametrize("ph,pw,h,w", [(24, 20, 104, 76), (48, 40, 208, 280), (24, 20, 16, 12), (138, 138, 550, 550)])
def test_checkerboard(ph, pw, h, w):
    proto, coef, box = checker_case(6, ph, pw, 4)
    for crop in (True, False):
        check(proto, coef, box, h, w, crop)


# ---- resize ratios -----------------------------------------------------------------------------------------------------
RESIZE = [
    (138, 138, 32, 1, 1, 12), (138, 138, 32, 1, 300, 12), (138, 138, 32, 300, 1, 12), (138, 138, 32, 5, 7, 12),
    (138, 138, 32, 64, 96, 12), (138, 138, 32, 137, 137, 12), (138, 138, 32, 139, 139, 12),
    (138, 138, 32, 203, 277, 12), (138, 138, 128, 550, 550, 8), (138, 138, 4, 1100, 1100, 3),
    (138, 138, 32, 2208, 1242, 3), (176, 176, 32, 700, 700, 6), (176, 176, 4, 480, 640, 6), (48, 40, 32, 203, 277, 12),
    (48, 40, 128, 1, 9, 12), (30, 1, 32, 97, 33, 12), (1, 30, 32, 33, 97, 12), (1, 1, 4, 9, 5, 4),
]


@pytest.mark.parametrize("ph,pw,k,h,w,n", RESIZE)
def test_resize_ratios(ph, pw, k, h, w, n):
    # the bound grows as k^2 against a value slope of sqrt(k): smaller boxes keep k = 128's undecided band near 1e-5
    proto, coef, box = random_case(ph * 7 + pw + h * 3 + w, n, ph, pw, k, 0.8 if k < 128 else 0.4)
    check(proto, coef, box, h, w)


# ---- band fallback and the shared-memory opt-in -----------------------------------------------------------------------
def mask_band(ph, pw, min_h, max_w):
    """mask.cu mask_band: rows per band, prototype rows per band and dynamic shared memory (a ColTab is 16 bytes)."""
    scale_h = f32(ph) / f32(min_h)
    band = 8
    while True:
        max_rows = int(float(band - 1) * float(scale_h)) + 4
        smem = max_w * 16 + max_rows * pw * 4
        if smem <= 200 * 1024 or band == 1:
            return band, max_rows, smem
        band //= 2


@pytest.mark.parametrize("h,w,band,opt_in", [(8, 9000, 4, True), (8, 12400, 1, True), (8, 11500, 2, True),
                                             (300, 3200, 8, True), (550, 550, 8, False)])
def test_band_fallback_and_shared_memory_opt_in(h, w, band, opt_in):
    assert mask_band(138, 138, h, w)[0] == band
    assert (mask_band(138, 138, h, w)[2] > 48 * 1024) == opt_in
    proto, coef, box = random_case(h + w, 4, 138, 138, 32)
    box[0] = [-0.1, -0.1, 1.1, 1.1]
    check(proto, coef, box, h, w)


# ---- groups and layout ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 8, 9, 100, 256])
def test_detection_groups(n):
    proto, coef, box = random_case(1000 + n, n, 138, 138, 32)
    check(proto, coef, box, 137, 203)


@pytest.mark.parametrize("fmt", FORMATS)
def test_batch_with_unaligned_image_planes(fmt):
    """yb_postprocess_batch, B = 3: with u8 and an odd h * w the per-image planes start at odd byte offsets."""
    from yolact_b200.output_utils import assemble_masks_batch
    B, n, h, w, ph, pw = 3, 5, 37, 51, 48, 40
    cases = [random_case(70 + b, n, ph, pw, 32) for b in range(B)]
    cases[1][2][0] = [np.nan, 0.2, 0.5, 0.6]
    proto, coef, box = (np.stack([c[i] for c in cases]) for i in range(3))
    plane = h * row_elems(fmt, w)
    buf = poisoned(fmt, GUARD + B * n * plane + GUARD)
    masks, boxes_px = assemble_masks_batch(cuda(proto), cuda(coef), cuda(box), h, w, True, fmt,
                                           masks_out=buf[GUARD:GUARD + B * n * plane].view(B, n, h, -1))
    torch.cuda.synchronize()
    assert_guard(buf, fmt, 0, GUARD, fmt)
    assert_guard(buf, fmt, GUARD + B * n * plane, buf.numel(), fmt)
    for b in range(B):
        v, e = R.mask_reference(proto[b], coef[b], box[b], h, w)
        judge(to_pixels(masks[b], fmt, h, w, "batch %s image %d" % (fmt, b)), v, e, "batch %s image %d" % (fmt, b))
        assert torch.equal(boxes_px[b], torch_boxes_px(box[b], h, w))


LIST_SIZES = [(3, 60, 80), (0, 20, 20), (4, 2, 9000), (5, 137, 139), (0, 1, 1), (1, 1, 1), (6, 33, 7)]


@pytest.mark.parametrize("fmt", FORMATS)
def test_list_with_caller_buffers(fmt):
    """yb_postprocess_list with every image's masks, pixel boxes and proto masks in caller buffers: the masks between
    guard bands of one buffer (each 16-byte aligned), n = 0 images included, and 1- and 2-row images beside a 9000-wide
    one, which drop the whole list to bands of 1 row."""
    ph, pw, k = 138, 138, 32
    assert mask_band(ph, pw, min(h for n, h, w in LIST_SIZES if n), max(w for n, h, w in LIST_SIZES if n))[0] == 1
    align = 16 // torch.tensor([], dtype=DTYPE[fmt]).element_size()
    offs, pos = [], GUARD
    for n, h, w in LIST_SIZES:
        offs.append(pos)
        pos += -(-(n * h * row_elems(fmt, w) + GUARD) // align) * align
    buf = poisoned(fmt, pos)
    dev = torch.device("cuda", torch.cuda.current_device())
    cases = [random_case(500 + i, n, ph, pw, k) for i, (n, h, w) in enumerate(LIST_SIZES)]
    cases[3][2][1] = [0.1, 0.2, np.nan, np.inf]
    total = sum(n for n, _, _ in LIST_SIZES)
    pm = torch.full((total + 1, ph, pw), float("nan"), device=dev)
    boxes_px = torch.full((total + 1, 4), -7, dtype=torch.int64, device=dev)
    keep, items, row = [], (_lib.YbPostItem * len(LIST_SIZES))(), 0
    for i, ((n, h, w), (proto, coef, box)) in enumerate(zip(LIST_SIZES, cases)):
        tp, tc, tb = cuda(proto), cuda(coef if n else np.zeros((1, k), f32)), cuda(box if n else np.zeros((1, 4), f32))
        keep += [tp, tc, tb]
        items[i] = _lib.YbPostItem(tp.data_ptr(), tc.data_ptr(), tb.data_ptr(), buf[offs[i]:].data_ptr(),
                                   boxes_px[row:].data_ptr(), pm[row:].data_ptr(), n, h, w)
        row += n
    _lib.check(_lib.load().yb_postprocess_list(_ops_handle(dev, k), items, len(LIST_SIZES), ph, pw, k, 1, FMT[fmt],
                                               _lib.current_stream(dev)), "yb_postprocess_list")
    torch.cuda.synchronize()
    assert_guard(buf, fmt, 0, GUARD, fmt)
    assert torch.equal(boxes_px[total], torch.full((4,), -7, dtype=torch.int64, device=dev))
    assert bool(pm[total].isnan().all())
    row = 0
    for i, ((n, h, w), (proto, coef, box)) in enumerate(zip(LIST_SIZES, cases)):
        end = offs[i] + n * h * row_elems(fmt, w)
        nxt = offs[i + 1] if i + 1 < len(offs) else buf.numel()
        assert_guard(buf, fmt, end, nxt, "list %s image %d" % (fmt, i))
        if n:
            what = "list %s image %d (%dx%d)" % (fmt, i, h, w)
            v, e = R.mask_reference(proto, coef, box, h, w)
            judge(to_pixels(buf[offs[i]:end].view(n, h, -1), fmt, h, w, what), v, e, what)
            assert torch.equal(boxes_px[row:row + n], torch_boxes_px(box, h, w)), what
            judge_proto_masks(pm[row:row + n], proto, coef, box, True, what)
        row += n


# ---- non-finite boxes --------------------------------------------------------------------------------------------------
NAN, INF = f32("nan"), f32("inf")


def nonfinite_boxes():
    base = np.array([0.2, 0.25, 0.7, 0.8], f32)
    boxes = [base.copy()]
    for i in range(4):                                     # NaN in each coordinate
        b = base.copy()
        b[i] = NAN
        boxes.append(b)
    for i, j in ((0, 2), (1, 3), (0, 1), (2, 3), (0, 3), (1, 2)):   # in pairs
        b = base.copy()
        b[[i, j]] = NAN
        boxes.append(b)
    boxes += [np.full(4, NAN, f32),
              [-INF, 0.25, 0.7, 0.8], [0.2, 0.25, INF, 0.8], [-INF, -INF, INF, INF], [INF, 0.25, 0.7, 0.8],
              [-INF, 0.25, NAN, 0.8], [0.2, -INF, 0.7, NAN],
              [-3e38, 0.25, 3e38, 0.8], [0.2, -3e38, 0.7, 3e38], [3e38, 0.25, 3e38, 0.8], [0.2, 0.25, 0.7, -3e38]]
    return np.array(boxes, f32)


@pytest.mark.parametrize("crop", [True, False])
@pytest.mark.parametrize("ph,pw,h,w", [(138, 138, 550, 550), (48, 40, 203, 277)])
def test_nonfinite_boxes(crop, ph, pw, h, w):
    box = nonfinite_boxes()
    cases = [saturated(11, len(box), ph, pw)] + ([random_case(12, len(box), ph, pw, 32)[:2]] if crop else [])
    for proto, coef in cases:
        v, _ = check(proto, coef, box, h, w, crop)
        if crop:
            nan = np.isnan(box).any(1)
            assert not (v[nan] > 0).any() and (v[~nan] > 0).any(axis=(1, 2)).sum() == 8
