"""The GPU path against the REAL reference's outputs at FULL size on the BASELINE.json configs
(tests/golden/full_*.npz: yolact_base@550 incl. a 640x480 postprocess target, yolact_plus_resnet50@550,
yolact_im700@700, yolact_plus_base@550), through the reference-facing API: net(x) in eval mode + postprocess().

  * f16x3 (the benched mode): north_star's bar -- class ids identical (ranks may swap only between scores closer than
    2e-5), boxes / scores within 1e-3, < 1e-3 mismatching mask pixels, raw heads within 2e-4.
  * f16tc (fast mode): reported, loosely bounded.
"""
import numpy as np
import pytest
import torch

import yolact_b200
from oracle.weights import deterministic_input, deterministic_state_dict
from tests.fullsize_golden import FULL_CASES, load_case, raw_errors
from tests.parity_utils import align
from yolact_b200.output_utils import postprocess

pytestmark = pytest.mark.gpu


def run_case(tag, precision):
    g, cfg, ref, (ph, pw) = load_case(tag)
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision=precision)
    net.detect.use_fast_nms = True                       # eval.py:871
    net.load_state_dict(deterministic_state_dict(net.state_dict(), int(g["seed"])))
    x = deterministic_input(1, int(g["size"]), int(g["size"]), int(g["seed_x"])).cuda()
    net.train()
    raw = {k: v.cpu().numpy() for k, v in net(x).items()}
    net.eval()
    preds = net(x)
    det = preds[0]["detection"]
    assert det is not None
    got = {"class": det["class"].cpu().numpy(), "score": det["score"].cpu().numpy(), "box": det["box"].cpu().numpy().copy()}
    classes, scores, boxes, masks = postprocess(preds, pw, ph, batch_idx=0)
    s2 = None
    if isinstance(scores, list):
        scores, s2 = scores
    got.update({"box_px": boxes.cpu().numpy(), "masks": masks.cpu().numpy() > 0.5,
                "score_maskiou": None if s2 is None else s2.cpu().numpy()})
    del net
    torch.cuda.empty_cache()
    return g, ref, got, raw_errors(raw, g)


@pytest.mark.parametrize("tag", FULL_CASES)
def test_benched_mode_vs_reference_at_full_size(tag):
    g, ref, got, e = run_case(tag, "f16x3")
    print(tag, "f16x3 raw errors", e)
    assert e["priors_equal"]
    for k in ("loc", "conf", "mask", "proto"):
        assert e[k] < 2e-4, (k, e[k])
    perm, ok = align(got, ref)
    assert ok, "class ids differ from the reference beyond score ties"
    strict = np.array_equal(got["class"], ref["class"])
    dbox = float(np.abs(got["box"][perm] - ref["box"]).max())
    dscore = float(np.abs(got["score"][perm] - ref["score"]).max())
    flips = float((got["masks"][perm] != ref["masks"]).mean())
    print(tag, "f16x3 strict class order %s, max dbox %.2e, max dscore %.2e, mask flips %.2e" % (strict, dbox, dscore, flips))
    assert dbox < 1e-3 and dscore < 1e-3                              # north_star: 1e-3 on boxes (and scores)
    assert np.abs(got["box_px"][perm] - ref["box_px"]).max() <= 1
    assert flips < 1e-3                                               # north_star: 1e-3 on masks
    if ref["score_maskiou"] is not None:
        assert np.abs(got["score_maskiou"][perm] - ref["score_maskiou"]).max() < 1e-3


@pytest.mark.parametrize("tag", ["full_base_550", "full_plus_base_550"])
def test_fast_mode_vs_reference_at_full_size(tag):
    g, ref, got, e = run_case(tag, "f16tc")
    perm, ok = align(got, ref)
    print(tag, "f16tc raw errors", e, "ranking equal mod ties:", ok, "reference detections found: %.3f" % float((perm >= 0).mean()))
    for k in ("loc", "conf", "proto"):
        assert e[k] < 5e-3, (k, e[k])
    assert e["mask"] < 4e-2
    assert (perm >= 0).mean() >= 0.85
