"""The oracle's Detect (oracle/yolact_oracle.detect_one) against the reference's own, at the parameter edges of
tests/golden/detect_edges.npz (oracle/gen_golden.py detect_edges): C = 2 / 21 / 96 / 129, top_k = 1 / 7 / 256,
max_dets = 1 / 100, nms_thresh = 0.3 / 0.5 / 0.7, conf_thresh = 0.05 / 0.5, mask_dim = 1 / 33, fast, cross-class and
traditional NMS, a batch whose middle image has no candidate, and NaN probabilities and boxes.  The GPU tests lean on
the oracle for the fixtures the golden is too small to hold, so it must be the reference's decision for decision."""
import numpy as np
import pytest

from oracle import yolact_oracle as O
from tests.conftest import load_golden

MODES = ("fast", "cc", "trad")


@pytest.fixture(scope="module")
def g():
    return load_golden("detect_edges")


def oracle(loc, conf, mask, priors, mode, top_k=200, max_dets=100, nms=0.5, conf_thresh=0.05):
    with np.errstate(invalid="ignore"):
        return O.detect_one(loc, conf, mask, priors, conf_thresh=conf_thresh, nms_thresh=nms, top_k=top_k,
                            max_dets=max_dets, cross_class=mode == "cc", traditional=mode == "trad", max_size=550)


def golden_priors(coef, mask):
    """The prior behind each golden row: its coefficient row is unique to one prior in these fixtures."""
    hit = np.all(coef[:, None, :] == mask[None, :, :coef.shape[1]], axis=2)
    assert (hit.sum(1) == 1).all()
    return hit.argmax(1)


def assert_matches(det, g, tag, b, loc, mask):
    """Decisions, scores and coefficients bit-exact; boxes bit-exact where loc[:, 2:] == 0 (expf(0) = 1, the rest is
    round-to-nearest), within 2 ulp elsewhere."""
    n = int(g[tag + "_counts"][b])
    if n == 0:
        assert det is None, (tag, b)
        return
    want = {k: g["%s_%d_%s" % (tag, b, k)] for k in ("box", "mask", "class", "score")}
    assert det["score"].shape[0] == n, (tag, b)
    assert np.array_equal(det["class"], want["class"]), (tag, b)
    assert np.array_equal(det["score"], want["score"]), (tag, b)
    assert np.array_equal(det["mask"], want["mask"]), (tag, b)
    box, ref = det["box"], want["box"]
    exact = np.all(loc[golden_priors(want["mask"], mask)][:, 2:] == 0, axis=1)
    assert np.array_equal(box[exact], ref[exact], equal_nan=True), (tag, b)
    assert np.array_equal(np.isnan(box), np.isnan(ref)), (tag, b)
    assert_box_ulps(box, ref, (tag, b))


def assert_box_ulps(box, ref, what, k=2):
    """|box - ref| <= k ulp of the box's largest coordinate: expf's error in w and h reaches every coordinate of the
    row through x1 = cx - w / 2 and x2 = x1 + w, whatever the coordinate's own magnitude."""
    ulp = np.spacing(np.nanmax(np.abs(ref), axis=1, keepdims=True)).astype(np.float64)
    ratio = np.abs(box.astype(np.float64) - ref) / ulp
    assert np.all((ratio <= k) | np.isnan(ref)), (what, float(np.nanmax(ratio)))


def test_golden_has_every_edge(g):
    cases = g["cases"]
    assert set(cases[:, 0]) == {2, 21, 96, 129}
    assert set(cases[:, 1]) == {0, 1, 2} and set(cases[:, 2]) == {1, 7, 256} and set(cases[:, 3]) == {1, 100}
    assert set(np.float32(cases[:, 4])) == {np.float32(0.3), np.float32(0.5), np.float32(0.7)}
    assert set(np.float32(cases[:, 5])) == {np.float32(0.05), np.float32(0.5)} and set(cases[:, 6]) == {1, 33}
    for i in range(len(cases)):
        assert g["case%d_counts" % i][1] == 0 and g["case%d_counts" % i][0] > 0     # the middle image is empty


@pytest.mark.parametrize("C", [2, 21, 96, 129])
def test_oracle_matches_reference_at_the_edges(g, C):
    loc, conf, mask, priors = (g["C%d_%s" % (C, k)] for k in ("loc", "conf", "mask", "priors"))
    ran = 0
    for i, row in enumerate(g["cases"]):
        if int(row[0]) != C:
            continue
        _, mode, top_k, max_dets, nms, conf_thresh, md = row
        for b in range(loc.shape[0]):
            det = oracle(loc[b], conf[b], mask[b][:, :int(md)], priors, MODES[int(mode)], top_k=int(top_k),
                                     max_dets=int(max_dets), nms=float(nms), conf_thresh=float(conf_thresh))
            assert_matches(det, g, "case%d" % i, b, loc[b], mask[b])
            ran += 1
    assert ran == 27


@pytest.mark.parametrize("mode", MODES)
def test_oracle_matches_reference_on_nan_inputs(g, mode):
    loc, conf, mask, priors = (g["nan_" + k] for k in ("loc", "conf", "mask", "priors"))
    det = oracle(loc[0], conf[0], mask[0], priors, mode)
    assert_matches(det, g, "nan_" + mode, 0, loc[0], mask[0])
    prior = golden_priors(det["mask"], mask[0])
    assert 5 not in prior and 6 not in prior      # a NaN foreground probability drops the prior
    s9, s12 = conf[0, 9, 3], conf[0, 12, 3]
    cls3 = det["class"] == 2
    if mode == "trad":
        # cython_nms: a NaN overlap is never >= thresh, so the NaN boxes neither suppress nor are suppressed
        assert 9 in prior and 12 in prior
        assert np.isnan(det["box"][prior == 9]).all()
    elif mode == "fast":
        # torch.max propagates NaN: the NaN box removes itself and every lower-scored box of its class
        assert not (cls3 & (det["score"] <= s9)).any() and (cls3 & (det["score"] > s9)).any()
    else:
        assert det["score"].min() > s9 and 12 not in prior
