"""CPU: the float64 mask reference (tests/mask_reference.py) that the GPU mask tests judge every pixel against.  Its
decided pixels must equal the oracle's fp32 masks and the reference's own golden masks, its undecided band must stay
thin, and its crop must empty a mask with a NaN box exactly as box_utils.crop does."""
import numpy as np
import pytest
import torch

from oracle import yolact_oracle as O
from tests import mask_reference as R
from tests.conftest import load_golden
from tests.helpers import unpack_masks

f32 = np.float32


def seeded(seed, n, ps=138, k=32):
    r = np.random.RandomState(seed)
    proto = np.maximum(r.standard_normal((ps, ps, k)), 0).astype(f32)
    coef = np.tanh(r.standard_normal((n, k))).astype(f32)
    c, wh = r.uniform(0.1, 0.9, (n, 2)), r.uniform(0.05, 0.6, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(f32)
    return proto, coef, box


def oracle_masks(proto, coef, box, h, w, crop):
    det = {"box": box, "mask": coef, "class": np.zeros(len(box), np.int64), "score": np.ones(len(box), f32),
           "proto": proto}
    return O.postprocess_one(det, w, h, crop_masks=crop)[3]


def test_decided_pixels_match_the_golden_and_the_oracle():
    g = load_golden("postprocess_unit")
    for (h, w) in ((550, 550), (203, 277), (64, 96)):
        for crop in (True, False):
            tag = "%dx%d_%s" % (h, w, "crop" if crop else "nocrop")
            v, e = R.mask_reference(g["proto"], g["coef"], g["box"], h, w, crop)
            dec, want = R.decide(v, e)
            assert (~dec).mean() <= 5e-5, tag   # 1.9e-5 uncropped at 550: the whole value surface is live
            for other in (unpack_masks(g["masks_" + tag], w), oracle_masks(g["proto"], g["coef"], g["box"], h, w, crop)):
                assert np.array_equal(other[dec] > 0.5, want[dec]), tag


@pytest.mark.parametrize("h,w", [(550, 550), (203, 277), (1100, 1100)])
def test_decided_pixels_match_the_oracle_on_seeded_cases(h, w):
    proto, coef, box = seeded(h * 7 + w, 12)
    box[3] = [-0.05, 0.3, 0.4, 1.1]
    v, e = R.mask_reference(proto, coef, box, h, w, True)
    dec, want = R.decide(v, e)
    assert (~dec).sum() <= 1e-5 * v.size, (~dec).sum()
    assert np.array_equal(oracle_masks(proto, coef, box, h, w, True)[dec] > 0.5, want[dec])
    assert 0.01 < want.mean() < 0.5


def test_proto_values_are_within_their_bound_of_the_oracle():
    proto, coef, box = seeded(3, 20, ps=69, k=128)
    val, bound, keep = R.proto_reference(proto, coef, box)
    pm = O.proto_masks(proto, coef, box).astype(np.float64)
    assert np.array_equal(pm != 0, keep & (val != 0))
    assert (np.abs(pm - val) <= bound).all()
    assert bound[keep].max() < 1e-4


def torch_crop_keep(box, h, w, padding=1):
    """box_utils.crop (box_utils.py:349-373) with sanitize_coordinates(cast=False) restated in torch: which positions
    of an all-ones [h, w, n] map survive."""
    boxes = torch.from_numpy(np.asarray(box, f32))

    def sanitize(a, b, size):
        a, b = a * size, b * size
        return torch.clamp(torch.min(a, b) - padding, min=0), torch.clamp(torch.max(a, b) + padding, max=size)

    n = boxes.shape[0]
    x1, x2 = sanitize(boxes[:, 0], boxes[:, 2], w)
    y1, y2 = sanitize(boxes[:, 1], boxes[:, 3], h)
    rows = torch.arange(w, dtype=x1.dtype).view(1, -1, 1).expand(h, w, n)
    cols = torch.arange(h, dtype=x1.dtype).view(-1, 1, 1).expand(h, w, n)
    keep = (rows >= x1.view(1, 1, -1)) * (rows < x2.view(1, 1, -1)) * (cols >= y1.view(1, 1, -1)) * \
        (cols < y2.view(1, 1, -1))
    return (torch.ones(h, w, n) * keep.float()).permute(2, 0, 1).numpy() > 0


NAN, INF = f32("nan"), f32("inf")
NONFINITE = np.array([[0.2, 0.2, 0.6, 0.6], [NAN, 0.2, 0.6, 0.6], [0.2, 0.2, NAN, 0.6], [NAN, NAN, NAN, NAN],
                      [-INF, 0.2, NAN, 0.6], [-INF, -INF, INF, INF], [0.2, NAN, 0.6, 0.6], [0.2, 0.2, 0.6, NAN],
                      [NAN, 0.2, NAN, 0.6], [0.2, NAN, 0.6, NAN], [INF, 0.2, 0.6, 0.6], [-3e38, 0.1, 3e38, 0.9],
                      [0.3, -3e38, 0.5, 3e38], [3e38, 0.1, 3e38, 0.9]], f32)


def test_nan_and_inf_boxes_crop_as_the_reference_does():
    keep = R.crop_keep(NONFINITE, 20, 20)
    assert np.array_equal(keep, torch_crop_keep(NONFINITE, 20, 20))
    assert keep[:6].sum((1, 2)).tolist() == [100, 0, 0, 0, 0, 400]
    # a NaN box leaves every pixel of the resized mask at 0 (decided); an overflowing product is a clamped edge
    v, e = R.mask_reference(np.full((20, 20, 4), 2, f32), np.ones((len(NONFINITE), 4), f32), NONFINITE, 45, 31)
    dec, want = R.decide(v, e)
    assert dec.all()
    nan_rows = np.isnan(NONFINITE).any(1)
    assert not want[nan_rows].any() and want[~nan_rows].any((1, 2)).all() == (keep[~nan_rows].any((1, 2))).all()
