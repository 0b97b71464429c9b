"""The implicit-GEMM convolution (tc_conv_kernel in f16tc / f16x3, the CUDA-core kernels in f16 / f32) through
yb_conv2d_ex, element by element against float64 at the edges of its tile, phase and channel arithmetic:

  a. M-tile edges: 3x3/s1/p1 and flattened 1x1 convolutions whose pixel counts sit below, at and above the 128-row
     tile, on one-pixel rows and columns;
  b. stride-2 phases: 3x3/s2/p1 and 1x1/s2/p0 on every map of sides 1..5 (a one-pixel side leaves a phase empty) and
     on long one-pixel rows and columns;
  c. K edges: one k-block, odd chunk counts and long rings (and a one-tile problem whose ring is one stage);
  d. N edges: output channel counts around every N tile width and the 64-channel staged-epilogue box, under every
     YB_CONV2D_BN, with a residual;
  e. the tilings (persistent grids, CTA pairs, two MMA warpgroups, PDL-friendly plans, stream-K) on edge shapes;
  f. locality: a NaN in one input element reaches exactly the outputs whose window covers it (and a NaN residual
     element exactly its own output); every other element is bitwise unchanged.  The half-precision encoders saturate
     a NaN operand to -65504 (DESIGN.md 3.1c), so there the outputs it reaches change instead of turning NaN;
  g. repeatability: the same call twice gives bitwise identical outputs in every tiling.

Every output is written between two guard bands that must come back unchanged, and every element is judged against
the per-element float64 bound of tests/conv_reference.py.
"""
import functools

import numpy as np
import pytest
import torch

from tests.conv_reference import (ACT_NONE, ACT_RELU, ACT_TANH, ROUNDED, act_f64, check, conv_ex_guarded, conv_f64,
                                  decode, f16, hd, he, out_hw, report_ratios, set_mode)  # noqa: F401

pytestmark = pytest.mark.gpu

ALL_PRECISIONS = ["f16tc", "f16x3", "f16", "f32"]     # the tensor-core modes need Cin % 64 == 0: every case here has it
TC_PRECISIONS = ["f16tc", "f16x3"]                     # the YB_CONV2D_* tilings only change the tensor-core plans

TILINGS = {
    "default": {},
    "grid3": {"YB_CONV2D_GRID": "3"},
    "pair": {"YB_CONV2D_PAIR": "1"},
    "pair_epi2": {"YB_CONV2D_PAIR": "1", "YB_CONV2D_EPI": "2"},
    "epi2": {"YB_CONV2D_EPI": "2"},
    "pdl": {"YB_CONV2D_PDL": "1"},
    "sk": {"YB_CONV2D_SK": "1"},
    "sk_grid5": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "5"},
    "sk_grid7_bn64": {"YB_CONV2D_SK": "1", "YB_CONV2D_GRID": "7", "YB_CONV2D_BN": "64"},
    "sk_pair": {"YB_CONV2D_SK": "1", "YB_CONV2D_PAIR": "1"},
}


def tilings_for(precision):
    # a PDL-friendly plan is single-pass only: the split mode would run its default plan again
    return [t for t in sorted(TILINGS) if not (t == "pdl" and precision == "f16x3")]


@functools.lru_cache(maxsize=32)
def problem(B, Cin, H, W, Cout, k, stride, pad, with_res):
    r = np.random.RandomState(B * 1000003 + Cin * 10007 + H * 101 + W * 7 + Cout * 3 + k + stride + pad)
    x = r.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = he(r, (Cout, Cin, k, k), Cin * k * k)
    bias = (r.standard_normal(Cout) * 0.1).astype(np.float32)
    Ho, Wo = out_hw(H, W, k, stride, pad)
    res = r.standard_normal((B, Cout, Ho, Wo)).astype(np.float32) if with_res else None
    return x, w, bias, res


@functools.lru_cache(maxsize=64)
def reference(B, Cin, H, W, Cout, k, stride, pad, with_res, rounded):
    """float64 conv + bias + residual (before the activation) and its scale, on the operands the mode consumes."""
    x, w, bias, res = problem(B, Cin, H, W, Cout, k, stride, pad, with_res)
    if rounded:
        x, w, res = f16(x), f16(w), f16(res)
    pre, scale = conv_f64(x, w, bias, stride, pad)
    if res is not None:
        rn = res.transpose(0, 2, 3, 1).astype(np.float64)
        pre, scale = pre + rn, scale + np.abs(rn)
    return pre, scale


def run_case(hd, B, Cin, H, W, Cout, k, stride, pad, precision, with_res=False, act=ACT_NONE, what=""):
    x, w, bias, res = problem(B, Cin, H, W, Cout, k, stride, pad, with_res)
    raw = conv_ex_guarded(hd, x, w, bias, res, stride, pad, act, precision)
    pre, scale = reference(B, Cin, H, W, Cout, k, stride, pad, with_res, precision in ROUNDED)
    check(decode(raw, precision, Cout), act_f64(pre, act), scale, precision,
          "%s %dx%dx%d Cin=%d Cout=%d %dx%d/s%d/p%d%s" % (what, B, H, W, Cin, Cout, k, k, stride, pad,
                                                          " +res" if with_res else ""))


# ----------------------------------------------------------------------------------------------------------------
# a. M-tile edges: pixel counts around the 128-row accumulator tile
# ----------------------------------------------------------------------------------------------------------------
M_SHAPES = [(1, 1, 1), (3, 1, 1), (1, 1, 130), (1, 130, 1), (2, 2, 3), (1, 11, 12), (2, 16, 8), (1, 129, 1),
            (5, 7, 9)]
# flattened 1x1: B * H * W = 1, 127, 128, 129, 255, 257, 128 * 132 + 1
FLAT_SHAPES = [(1, 1, 1), (1, 1, 127), (2, 8, 8), (3, 43, 1), (3, 5, 17), (1, 1, 257), (1, 61, 277)]


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("B,H,W", M_SHAPES, ids=lambda v: str(v))
def test_a_m_tile_edges_3x3(hd, B, H, W, precision):
    run_case(hd, B, 64, H, W, 64, 3, 1, 1, precision, what="M edge")


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("B,H,W", sorted(set(M_SHAPES + FLAT_SHAPES)), ids=lambda v: str(v))
def test_a_m_tile_edges_flat_1x1(hd, B, H, W, precision):
    run_case(hd, B, 64, H, W, 64, 1, 1, 0, precision, what="M edge")


# ----------------------------------------------------------------------------------------------------------------
# b. stride-2 phases: every map with sides 1..5 (H == 1 or W == 1 leaves the odd phase of a 3x3/s2/p1 conv empty)
# ----------------------------------------------------------------------------------------------------------------
S2_SHAPES = [(h, w) for h in range(1, 6) for w in range(1, 6)] + [(1, 257), (257, 1), (69, 69)]


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("H,W", S2_SHAPES, ids=lambda v: str(v))
def test_b_stride2_phases_3x3(hd, H, W, precision):
    run_case(hd, 2, 64, H, W, 64, 3, 2, 1, precision, what="s2 phase")


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("H,W", S2_SHAPES, ids=lambda v: str(v))
def test_b_stride2_phases_1x1(hd, H, W, precision):
    run_case(hd, 2, 64, H, W, 64, 1, 2, 0, precision, what="s2 phase")


# ----------------------------------------------------------------------------------------------------------------
# c. K edges: one k-block, odd chunk counts, long rings
# ----------------------------------------------------------------------------------------------------------------
K_CASES = [(1, c) for c in (64, 128, 192, 320, 2048)] + [(3, c) for c in (64, 192, 512)]


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
@pytest.mark.parametrize("k,Cin", K_CASES, ids=lambda v: str(v))
def test_c_k_edges(hd, k, Cin, precision):
    run_case(hd, 2, Cin, 13, 11, 64, k, 1, k // 2, precision, what="K edge")


@pytest.mark.parametrize("precision", ALL_PRECISIONS)
def test_c_one_tile_one_stage(hd, precision):
    """64 pixels x one 64-channel k-block: one tile of one k-block, the plan's ring is one stage deep."""
    run_case(hd, 1, 64, 8, 8, 64, 1, 1, 0, precision, what="one stage")


# ----------------------------------------------------------------------------------------------------------------
# d. N edges: every N tile width, the staged (64-channel box) and direct epilogues, partial last N tiles
# ----------------------------------------------------------------------------------------------------------------
COUTS = [1, 7, 8, 12, 27, 32, 63, 64, 65, 72, 127, 128, 129, 243, 256, 257]
BNS = {"bn32": "32", "bn64": "64", "bn128": "128", "bn256": "256"}


@pytest.mark.parametrize("bn", sorted(BNS))
@pytest.mark.parametrize("precision", TC_PRECISIONS)
@pytest.mark.parametrize("Cout", COUTS)
def test_d_n_edges(hd, Cout, precision, bn, monkeypatch):
    set_mode(monkeypatch, {"YB_CONV2D_BN": BNS[bn]})
    run_case(hd, 2, 64, 9, 10, Cout, 3, 1, 1, precision, with_res=True, act=ACT_RELU, what="N edge " + bn)


@pytest.mark.parametrize("precision", ["f16", "f32"])
@pytest.mark.parametrize("Cout", COUTS)
def test_d_n_edges_cuda_cores(hd, Cout, precision):
    run_case(hd, 2, 64, 9, 10, Cout, 3, 1, 1, precision, with_res=True, act=ACT_RELU, what="N edge")


# ----------------------------------------------------------------------------------------------------------------
# e. tilings, on edge shapes; a 1x1 residual under EPI=2 in f16x3 is read straight from global memory (res_direct)
# ----------------------------------------------------------------------------------------------------------------
TILING_SHAPES = {   # B, Cin, H, W, Cout, k, stride, pad, with_res, act
    "3x3-132px": (1, 64, 11, 12, 64, 3, 1, 1, False, ACT_NONE),
    "3x3s2-Co72": (2, 128, 13, 11, 72, 3, 2, 1, False, ACT_RELU),
    "1x1-129px-res": (1, 192, 3, 43, 128, 1, 1, 0, True, ACT_RELU),
    "1x1-315px-Co256-res": (5, 64, 7, 9, 256, 1, 1, 0, True, ACT_NONE),
    "3x3-5x5-res": (3, 256, 5, 5, 64, 3, 1, 1, True, ACT_RELU),
    "1x1s2-9x9": (2, 128, 9, 9, 128, 1, 2, 0, False, ACT_NONE),
}


@pytest.mark.parametrize("shape", sorted(TILING_SHAPES))
@pytest.mark.parametrize("precision,tiling", [(p, t) for p in TC_PRECISIONS for t in tilings_for(p)],
                         ids=lambda v: str(v))
def test_e_tilings(hd, precision, tiling, shape, monkeypatch):
    set_mode(monkeypatch, TILINGS[tiling])
    B, Cin, H, W, Cout, k, s, p, with_res, act = TILING_SHAPES[shape]
    run_case(hd, B, Cin, H, W, Cout, k, s, p, precision, with_res=with_res, act=act, what=tiling)


# ----------------------------------------------------------------------------------------------------------------
# f. locality: one NaN input (or residual) element reaches exactly the outputs that read it
# ----------------------------------------------------------------------------------------------------------------
def element_bits(raw, precision, Cp):
    """The raw output as bit patterns [B, Ho, Wo, Cp, planes] (a split pair's hi and lo side by side)."""
    if raw.dtype == torch.float32:
        return raw.view(torch.int32).cpu().numpy()[..., :Cp, None]
    bits = raw.view(torch.int16).cpu().numpy()
    if precision == "f16x3":
        return np.stack([bits[..., :Cp], bits[..., Cp:2 * Cp]], -1)
    return bits[..., :Cp, None]


def covering(n_out, i, k, stride, pad):
    """Output indices whose k-wide window at this stride and pad covers input index i."""
    return np.array([o * stride - pad <= i <= o * stride - pad + k - 1 for o in range(n_out)])


def probe_pixels(B, H, W, r):
    """Every pixel of a small map; the corners, edge midpoints and a few seeded pixels of a larger one."""
    if B * H * W <= 40:
        return [(b, i, j) for b in range(B) for i in range(H) for j in range(W)]
    pts = {(b, i, j) for b in (0, B - 1) for i in (0, H // 2, H - 1) for j in (0, W // 2, W - 1)}
    pts |= {(int(r.randint(B)), int(r.randint(H)), int(r.randint(W))) for _ in range(4)}
    return sorted(pts)


LOCALITY_GEOMETRIES = {   # B, H, W, k, stride, pad, act
    "s1-small": (2, 4, 5, 3, 1, 1, ACT_NONE),
    "s2-small": (2, 5, 4, 3, 2, 1, ACT_TANH),
    "s1-large": (2, 23, 19, 3, 1, 1, ACT_TANH),
    "s2-large": (1, 30, 27, 3, 2, 1, ACT_NONE),
}
LOCALITY_RUNS = [(p, t) for p in TC_PRECISIONS for t in ("default", "pair", "sk")] + [("f32", "default")]
CIN_L, COUT_L = 64, 64


@pytest.mark.parametrize("geometry", sorted(LOCALITY_GEOMETRIES))
@pytest.mark.parametrize("precision,tiling", LOCALITY_RUNS, ids=lambda v: str(v))
def test_f_locality_nan_input(hd, precision, tiling, geometry, monkeypatch):
    set_mode(monkeypatch, TILINGS[tiling])
    B, H, W, k, s, p, act = LOCALITY_GEOMETRIES[geometry]
    x, w, bias, _ = problem(B, CIN_L, H, W, COUT_L, k, s, p, False)
    x = x * np.float32(0.25)   # |conv| well below 4: no clean tanh output rounds to +-1 in fp16 and hides a change
    Ho, Wo = out_hw(H, W, k, s, p)
    clean = conv_ex_guarded(hd, x, w, bias, None, s, p, act, precision)
    clean_bits = element_bits(clean, precision, COUT_L)
    assert np.isfinite(decode(clean, precision, COUT_L)).all()
    r = np.random.RandomState(H * W)
    for b, i, j in probe_pixels(B, H, W, r):
        c = (7 * i + 3 * j + b) % CIN_L
        xn = x.copy()
        xn[b, c, i, j] = np.nan
        y = conv_ex_guarded(hd, xn, w, bias, None, s, p, act, precision)
        want = np.zeros((B, Ho, Wo), bool)
        want[b] = covering(Ho, i, k, s, p)[:, None] & covering(Wo, j, k, s, p)[None, :]
        changed = (element_bits(y, precision, COUT_L) != clean_bits).any(-1)
        reached = np.isnan(decode(y, precision, COUT_L)) if precision == "f32" else changed
        where = "NaN at input (%d, %d, %d, %d)" % (b, c, i, j)
        assert reached[want].all(), "%s: %d outputs it reaches are unchanged" % (where, (~reached[want]).sum())
        assert not changed[~want].any(), "%s: %d outputs it does not reach changed, first at %s" % (
            where, changed[~want].sum(), tuple(np.argwhere(changed & ~want[..., None])[0]))


@pytest.mark.parametrize("geometry", ["s1-small", "s2-large"])
@pytest.mark.parametrize("precision,tiling", LOCALITY_RUNS, ids=lambda v: str(v))
def test_f_locality_nan_residual(hd, precision, tiling, geometry, monkeypatch):
    set_mode(monkeypatch, TILINGS[tiling])
    B, H, W, k, s, p, act = LOCALITY_GEOMETRIES[geometry]
    x, w, bias, res = problem(B, CIN_L, H, W, COUT_L, k, s, p, True)
    Ho, Wo = out_hw(H, W, k, s, p)
    clean_bits = element_bits(conv_ex_guarded(hd, x, w, bias, res, s, p, act, precision), precision, COUT_L)
    r = np.random.RandomState(Ho * Wo)
    for b, i, j in probe_pixels(B, Ho, Wo, r)[::3]:
        c = (5 * i + 11 * j + b) % COUT_L
        rn = res.copy()
        rn[b, c, i, j] = np.nan
        y = conv_ex_guarded(hd, x, w, bias, rn, s, p, act, precision)
        changed = (element_bits(y, precision, COUT_L) != clean_bits).any(-1)
        assert changed[b, i, j, c] and (precision != "f32" or np.isnan(decode(y, precision, COUT_L)[b, i, j, c]))
        changed[b, i, j, c] = False
        assert not changed.any(), "NaN residual at (%d, %d, %d, %d): %d other outputs changed" % (
            b, c, i, j, changed.sum())


# ----------------------------------------------------------------------------------------------------------------
# g. repeatability: the plan's summation order does not change from one call to the next
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", sorted(TILING_SHAPES))
@pytest.mark.parametrize("precision,tiling", [(p, t) for p in TC_PRECISIONS for t in tilings_for(p)],
                         ids=lambda v: str(v))
def test_g_repeatable(hd, precision, tiling, shape, monkeypatch):
    set_mode(monkeypatch, TILINGS[tiling])
    B, Cin, H, W, Cout, k, s, p, with_res, act = TILING_SHAPES[shape]
    x, w, bias, res = problem(B, Cin, H, W, Cout, k, s, p, with_res)
    a = conv_ex_guarded(hd, x, w, bias, res, s, p, act, precision)
    b = conv_ex_guarded(hd, x, w, bias, res, s, p, act, precision)
    bits = torch.int32 if a.dtype == torch.float32 else torch.int16
    assert torch.equal(a.view(bits), b.view(bits))
