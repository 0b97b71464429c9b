"""The references the DCNv2 GPU tests compare against, checked on the CPU: the float64 path of the vectorised oracle
against the reference's golden case, the vectorised oracle against a scalar restatement written separately, and the
probe cases' own premise (every probe offset reaches its target position exactly in fp32)."""
import numpy as np
import pytest

from oracle import yolact_oracle as O
from tests.conftest import load_golden
from tests.dcn_probe import GEOMETRIES, axis_expectation, build_probe_case, out_hw, selected_columns

f32 = np.float32


# ----------------------------------------------------------------------------------------------------------------
# Scalar restatement, one (pixel, tap, channel) at a time, of modulated_deformable_im2col_gpu_kernel and
# dmcn_im2col_bilinear (external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:151-189 and :25-54).  Every value is an
# np.float32 scalar, so every operation rounds to fp32 like the reference's `float`.
# ----------------------------------------------------------------------------------------------------------------
def naive_bilinear(img, height, width, h, w):
    h_low = int(np.floor(h))
    w_low = int(np.floor(w))
    h_high = h_low + 1
    w_high = w_low + 1
    lh = h - f32(h_low)
    lw = w - f32(w_low)
    hh, hw = f32(1) - lh, f32(1) - lw
    v1 = v2 = v3 = v4 = f32(0)
    if h_low >= 0 and w_low >= 0:
        v1 = img[h_low, w_low]
    if h_low >= 0 and w_high <= width - 1:
        v2 = img[h_low, w_high]
    if h_high <= height - 1 and w_low >= 0:
        v3 = img[h_high, w_low]
    if h_high <= height - 1 and w_high <= width - 1:
        v4 = img[h_high, w_high]
    w1, w2, w3, w4 = hh * hw, hh * lw, lh * hw, lh * lw
    return w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4


def naive_column(x, offset, mask, b, c, tap, h_col, w_col, stride, pad, dil):
    height, width = x.shape[2:]
    i, j = divmod(tap, 3)
    h_in = h_col * stride - pad
    w_in = w_col * stride - pad
    offset_h = offset[b, 2 * tap, h_col, w_col]
    offset_w = offset[b, 2 * tap + 1, h_col, w_col]
    val = f32(0)
    with np.errstate(over="ignore", invalid="ignore"):
        h_im = f32(h_in + i * dil) + offset_h
        w_im = f32(w_in + j * dil) + offset_w
    if h_im > -1 and w_im > -1 and h_im < height and w_im < width:
        val = naive_bilinear(x[b, c], height, width, h_im, w_im)
    return val * mask[b, tap, h_col, w_col]


def naive_selected_columns(case):
    x, offset, mask = case["x"], case["offset"], case["mask"]
    B, _, Ho, Wo = mask.shape
    out = np.zeros((B, len(case["sel"]), Ho, Wo), f32)
    for b in range(B):
        for o, (tap, c) in enumerate(case["sel"]):
            for ho in range(Ho):
                for wo in range(Wo):
                    out[b, o, ho, wo] = naive_column(x, offset, mask, b, c, tap, ho, wo, case["stride"], case["pad"],
                                                     case["dil"])
    return out


@pytest.fixture(scope="module", params=GEOMETRIES, ids=lambda g: "s%d-p%d-d%d-%dx%d" % g)
def case(request):
    s, pad, dil, H, W = request.param
    return build_probe_case(H, W, s, pad, dil, 64, seed=100 * H + 10 * s + pad)


def test_probe_offsets_reach_their_targets_exactly(case):
    """base + offset == target in fp32 for every probe; the far and non-finite offsets land outside the image."""
    H, W = case["x"].shape[2:]
    h_im, w_im, valid = O.dcn_v2_positions(case["offset"], H, W, case["stride"], case["pad"], case["dil"])
    kinds = set()
    for p in case["probes"]:
        at = (p["b"], p["tap"], p["ho"], p["wo"])
        for axis, pos in (("h", h_im[at]), ("w", w_im[at])):
            if p[axis] is None:
                continue
            name, target = p[axis]
            kinds.add((axis, name))
            if name == "far":
                assert not valid[at] and not (-1 < pos < max(H, W))
            else:
                assert pos == target and pos.dtype == f32, (p, pos)
    assert len(kinds) == 22   # ten positions and the far offsets, on both axes


def test_vectorised_oracle_equals_scalar_restatement_bitwise(case):
    cols = O.dcn_v2_columns(case["x"], case["offset"], case["mask"], case["stride"], case["pad"], case["dil"])
    assert cols.dtype == f32
    got, want = selected_columns(cols, case), naive_selected_columns(case)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # float64 blend of the same corners: within a few fp32 roundings of the blend's magnitude
    c64, mag = O.dcn_v2_columns(case["x"], case["offset"], case["mask"], case["stride"], case["pad"], case["dil"],
                                acc=np.float64, with_abs=True)
    assert c64.dtype == np.float64 and np.isfinite(c64).all()
    assert (np.abs(selected_columns(c64, case) - want) <= 2.0 ** -21 * selected_columns(mag, case)).all()


def test_probe_positions_give_the_tabulated_samples(case):
    """Integral position: the pixel itself (at n-1 the far corners do not exist); -1 and n: 0; -0.5 and n-0.5: half
    of the border pixel; far and non-finite offsets: 0 -- read off the scalar restatement."""
    x, mask = case["x"], case["mask"]
    H, W = x.shape[2:]
    checked = 0
    for p in case["probes"]:
        if p["h"] is None or p["w"] is None:
            continue
        b, tap, ho, wo = p["b"], p["tap"], p["ho"], p["wo"]
        far = "far" in (p["h"][0], p["w"][0])
        if not far and ("ulp" in p["h"][0] or "ulp" in p["w"][0]):
            continue
        eh = None if far else axis_expectation(p["h"][0], H)
        ew = None if far else axis_expectation(p["w"][0], W)
        for c in case["sel_c"]:
            got = naive_column(x, case["offset"], mask, b, c, tap, ho, wo, case["stride"], case["pad"], case["dil"])
            if eh is None or ew is None:
                assert got == 0
            else:
                want = np.float64(eh[1] * ew[1]) * x[b, c, eh[0], ew[0]] * mask[b, tap, ho, wo]
                assert abs(got - want) <= 2.0 ** -22 * abs(want)
        checked += 1
    assert checked == 43   # 6 x 6 tabulated positions in both axes, 7 far offsets


def test_one_ulp_inside_the_border_is_inside():
    """nextafter(-1, 0) and nextafter(n, 0) pass the inside test and sample the one row of corners that exists, with
    the tiny weight the fraction leaves it: 2^-24 of row 0, and 2^-22 (n = 4) of row n-1."""
    x = np.zeros((1, 1, 4, 4), f32)
    x[0, 0, 0, :] = 3.0
    x[0, 0, 3, :] = 5.0
    off = np.zeros((1, 18, 4, 4), f32)
    m = np.ones((1, 9, 4, 4), f32)
    lo, hi = np.nextafter(f32(-1), f32(0)), np.nextafter(f32(4), f32(0))
    off[0, 2, 1, 1] = lo               # tap 1 of pixel (1, 1), pad 1: base row 0
    off[0, 8, 2, 2] = hi - f32(2)      # tap 4 of pixel (2, 2): base row 2
    cols = O.dcn_v2_columns(x, off, m, 1, 1, 1, acc=np.float64)
    assert cols[0, 0, 1, 1, 1] == 3.0 * 2.0 ** -24
    assert cols[0, 0, 4, 2, 2] == 5.0 * 2.0 ** -22
    assert naive_column(x, off, m, 0, 0, 4, 2, 2, 1, 1, 1) == f32(5.0 * 2.0 ** -22)
    assert naive_column(x, off, m, 0, 0, 1, 1, 1, 1, 1, 1) == f32(3.0 * 2.0 ** -24)


@pytest.mark.parametrize("tag", ["s1", "s2"])
def test_float64_path_against_reference_golden(tag):
    g = load_golden("dcn_unit")
    args = (g[tag + "_x"], g[tag + "_offset"], g[tag + "_mask"], g[tag + "_w"], g[tag + "_bias"], int(g[tag + "_stride"]), 1, 1)
    y64 = O.dcn_v2_forward(*args, acc=np.float64)
    assert y64.dtype == np.float64
    assert np.abs(y64 - g[tag + "_y"]).max() <= 2e-5
    y32 = O.dcn_v2_forward(*args)
    assert y32.dtype == f32 and np.abs(y32 - y64).max() <= 2e-5


def test_columns_then_contraction_is_the_forward():
    r = np.random.RandomState(3)
    x = r.standard_normal((2, 16, 9, 8)).astype(f32)
    Ho, Wo = out_hw(9, 8, 2, 2, 2)
    off = (r.standard_normal((2, 18, Ho, Wo)) * 2).astype(f32)
    m = r.uniform(size=(2, 9, Ho, Wo)).astype(f32)
    w = r.standard_normal((5, 16, 3, 3)).astype(f32)
    bias = r.standard_normal(5).astype(f32)
    y = O.dcn_v2_forward(x, off, m, w, bias, 2, 2, 2)
    cols = O.dcn_v2_columns(x, off, m, 2, 2, 2)
    assert cols.shape == (2, 16, 9, Ho, Wo)
    assert np.array_equal(y, O.dcn_v2_contract(cols, w, bias))
