"""Whole path through the reference-facing API (yolact_b200.Yolact / postprocess) against the
reference's golden outputs.

  * precision='f16x3' (split-precision tensor-core, the default and benched mode) and precision='f32' (fp32 CUDA-core
    second opinion): raw head tensors within 1e-4 of the reference, class ids bit-exact, boxes/scores within 2e-5
    (north_star asks for 1e-3), binarised masks < 1e-3 mismatching pixels.
  * precision='f16tc' (single-pass fp16 tensor-core, the fast mode): fp16 operands, fp32 accumulation.  Tolerances are
    written next to each assert; discrete outputs (class ids, NMS keep set) are reported as agreement
    ratios because they are discontinuous in the scores (SURVEY.md section 7, hard part 1).
"""
import numpy as np
import pytest
import torch

import yolact_b200
from oracle import yolact_oracle as O
from oracle.weights import deterministic_state_dict, deterministic_input
from tests.conftest import load_golden
from tests.helpers import cfg_for, unpack_masks, rel_err
from tests.parity_utils import align
from yolact_b200.output_utils import postprocess

pytestmark = pytest.mark.gpu

NET_CASES = ["net_resnet50_160", "net_base_192x160_b2", "net_plus_resnet50_256", "net_darknet53_160"]
_cache = {}


def build(case, precision):
    key = (case, precision)
    if key not in _cache:
        g = load_golden(case)
        cfg = cfg_for(str(g["config"]))
        yolact_b200.cfg.replace(cfg.copy())
        net = yolact_b200.Yolact(cfg, precision=precision)
        net.detect.use_fast_nms = True   # what eval.py does from --fast_nms (default True, eval.py:50,871)
        net.load_state_dict(deterministic_state_dict(net.state_dict(), int(g["seed"])))
        _cache[key] = (g, cfg, net)
    g, cfg, net = _cache[key]
    yolact_b200.cfg.replace(cfg.copy())
    return g, cfg, net


EXACT_MODES = ["f16x3", "f32"]
# f32 (CUDA-core FMA) and f16x3 (split-precision tensor cores: each MMA pass accumulates with the tensor core's own fp32
# rounding) both sit far inside these bounds; north_star asks for 1e-3.
RAW_TOL = {"f32": 1e-4, "f16x3": 2e-4}
DET_ATOL = {"f32": 2e-5, "f16x3": 2e-4}


@pytest.mark.parametrize("prec", EXACT_MODES)
@pytest.mark.parametrize("case", NET_CASES)
def test_raw_heads_exact_modes(case, prec):
    g, cfg, net = build(case, prec)
    net.train()
    out = net(torch.from_numpy(g["x"]).cuda())
    rs = int(g["row_stride"])
    assert np.array_equal(out["priors"].cpu().numpy(), g["raw_priors"])           # priors: bit-exact
    for k in ("proto", "loc", "conf", "mask"):
        got = out[k].cpu().numpy()
        if k != "proto":
            got = got[:, ::rs]
        e = rel_err(got, g["raw_" + k])
        print(case, prec, k, "rel err %.2e" % e)
        assert e < RAW_TOL[prec], (k, e)


@pytest.mark.parametrize("case", NET_CASES)
def test_raw_heads_f16tc_mode(case):
    g, cfg, net = build(case, "f16tc")
    net.train()
    out = net(torch.from_numpy(g["x"]).cuda())
    rs = int(g["row_stride"])
    assert np.array_equal(out["priors"].cpu().numpy(), g["raw_priors"])
    # fp16 operands (rel 2^-11 per rounding) through up to ~100 layers: allow 1.5e-2 of the tensor's range
    for k in ("proto", "loc", "conf", "mask"):
        got = out[k].cpu().numpy()
        if k != "proto":
            got = got[:, ::rs]
        assert np.isfinite(got).all()
        e = rel_err(got, g["raw_" + k])
        print(case, "f16tc", k, "rel err %.2e" % e)
        assert e < 1.5e-2, (k, e)


@pytest.mark.parametrize("prec", EXACT_MODES)
@pytest.mark.parametrize("case", ["net_resnet50_160", "net_base_192x160_b2", "net_plus_resnet50_256"])
def test_backbone_features_exact_modes(case, prec):
    g, cfg, net = build(case, prec)
    net.train()
    net(torch.from_numpy(g["x"]).cuda())
    for i in range(4):
        f = net.debug_feature(i, torch.device("cuda", 0)).cpu().numpy()
        e = rel_err(f[:, ::7, ::3, ::3], g["feat_c%d_sample" % i])
        assert e < 1e-4, (i, e)


@pytest.mark.parametrize("prec", EXACT_MODES)
@pytest.mark.parametrize("case", NET_CASES)
def test_eval_pipeline_exact_modes(case, prec):
    """net(x) in eval mode + postprocess: the exact call sequence of eval.py (eval.py:949,266)."""
    g, cfg, net = build(case, prec)
    net.eval()
    preds = net(torch.from_numpy(g["x"]).cuda())
    ph, pw = (int(v) for v in g["post_hw"])
    assert len(preds) == g["x"].shape[0]
    for b, p in enumerate(preds):
        det = p["detection"]
        assert p["net"] is net and det is not None
        n = int(g["det_counts"][b])
        assert det["score"].shape[0] == n
        # class ids: identical, rank for rank; ranks may swap only between reference scores closer than 2e-5 (ties at
        # the resolution of ANY fp32 implementation -- tests/parity_utils.align)
        got = {"class": det["class"].cpu().numpy(), "score": det["score"].cpu().numpy(), "box": det["box"].cpu().numpy()}
        ref_det = {"class": g["det%d_class" % b], "score": g["det%d_score" % b], "box": g["det%d_box" % b]}
        perm, ok = align(got, ref_det)
        assert ok, "class ids differ from the reference beyond score ties"
        if prec == "f32":
            assert np.array_equal(got["class"], ref_det["class"])
        tol = DET_ATOL[prec]
        np.testing.assert_allclose(got["score"][perm], ref_det["score"], atol=tol)
        np.testing.assert_allclose(got["box"][perm], ref_det["box"], atol=tol)
        np.testing.assert_allclose(det["mask"].cpu().numpy()[perm], g["det%d_mask" % b], atol=tol)
        classes, scores, boxes, masks = postprocess(preds, pw, ph, batch_idx=b)
        if isinstance(scores, list):                                               # YOLACT++ (output_utils.py:84-88)
            np.testing.assert_allclose(scores[1].cpu().numpy()[perm], g["post%d_scores_maskiou" % b], rtol=1e-3, atol=10 * tol)
            scores = scores[0]
        assert np.array_equal(classes.cpu().numpy()[perm], g["post%d_classes" % b])
        assert np.abs(boxes.cpu().numpy()[perm] - g["post%d_boxes" % b]).max() <= 1  # .long() of x*w at 1e-5 noise
        ref = unpack_masks(g["post%d_masks_packed" % b], pw)
        mism = float((masks.cpu().numpy()[perm] != ref).mean())
        print(case, prec, "image", b, "mask pixel mismatch %.2e" % mism)
        assert mism < 1e-3


@pytest.mark.parametrize("case", NET_CASES)
def test_eval_pipeline_f16tc_mode_agreement(case):
    g, cfg, net = build(case, "f16tc")
    net.eval()
    preds = net(torch.from_numpy(g["x"]).cuda())
    ph, pw = (int(v) for v in g["post_hw"])
    for b, p in enumerate(preds):
        det = p["detection"]
        assert det is not None
        gb, gc, gs = g["det%d_box" % b], g["det%d_class" % b], g["det%d_score" % b]
        box, cls, sc = det["box"].cpu().numpy(), det["class"].cpu().numpy(), det["score"].cpu().numpy()
        # match detections by (class, IoU > 0.9): order may differ where scores are within fp16 noise
        matched, max_box, max_score = 0, 0.0, 0.0
        for i in range(len(gs)):
            cand = np.nonzero(cls == gc[i])[0]
            if cand.size == 0:
                continue
            d = np.abs(box[cand] - gb[i]).max(axis=1)
            j = cand[d.argmin()]
            if d.min() < 2e-2:
                matched += 1
                max_box = max(max_box, float(d.min()))
                max_score = max(max_score, float(abs(sc[j] - gs[i])))
        frac = matched / float(len(gs))
        print(case, "image", b, "f16tc matched %.3f  max box delta %.2e  max score delta %.2e" % (frac, max_box, max_score))
        assert frac >= 0.85
        classes, scores, boxes, masks = postprocess(preds, pw, ph, batch_idx=b)
        assert masks.shape[1:] == (ph, pw) and set(np.unique(masks.cpu().numpy())) <= {0.0, 1.0}


def test_full_size_yolact_base_f16tc_vs_f32_and_oracle():
    """BASELINE configs[1] shape: yolact_base @550 (B=2 here to bound CPU time).  GPU fp32 mode is the
    second opinion for the tensor-core mode; the CPU oracle checks image 0."""
    cfg = cfg_for("yolact_base_config")
    yolact_b200.cfg.replace(cfg.copy())
    x = deterministic_input(2, 550, 550, 99)
    outs = {}
    for prec in ("f32", "f16tc", "f16x3"):
        net = yolact_b200.Yolact(cfg, precision=prec)
        net.detect.use_fast_nms = True   # what eval.py does from --fast_nms (default True, eval.py:50,871)
        sd = deterministic_state_dict(net.state_dict(), 1)
        net.load_state_dict(sd)
        net.train()
        outs[prec] = {k: v.cpu() for k, v in net(x.cuda()).items()}
        assert outs[prec]["loc"].shape == (2, 19248, 4) and outs[prec]["proto"].shape == (2, 138, 138, 32)
        del net
        torch.cuda.empty_cache()
    for k in ("loc", "conf", "mask", "proto"):
        e = rel_err(outs["f16tc"][k].numpy(), outs["f32"][k].numpy())
        print("yolact_base@550 f16tc vs f32", k, "rel err %.2e" % e)
        # tanh-ed coefficients of 19248 priors: the max over 1.2M values of an fp16-operand K=2304 dot
        assert e < (4e-2 if k == "mask" else 1.5e-2)
    orc = O.ConvStackOracle(cfg, sd)
    ref = orc.forward(x[:1])
    for prec in ("f32", "f16x3"):
        for k in ("loc", "conf", "mask", "proto"):
            e = rel_err(outs[prec][k][:1].numpy(), ref[k].numpy())
            print("yolact_base@550 %s vs CPU oracle" % prec, k, "rel err %.2e" % e)
            assert e < RAW_TOL[prec] * 2
    assert np.array_equal(outs["f32"]["priors"].numpy(), ref["priors"].numpy())


def test_graph_replay_is_deterministic_and_batch_independent():
    g, cfg, net = build("net_resnet50_160", "f16tc")
    net.eval()
    x = torch.from_numpy(g["x"]).cuda()
    a = net.infer_padded(x)
    b = net.infer_padded(x)      # second call captures the CUDA graph
    c = net.infer_padded(x)      # third call replays it
    torch.cuda.synchronize()
    for t0, t1, t2 in zip(a[:5], b[:5], c[:5]):
        assert torch.equal(t0, t1) and torch.equal(t0, t2)
    # images are independent: a batch of two copies gives the single-image result twice
    x2 = torch.cat([x, x], 0)
    d = net.infer_padded(x2)
    torch.cuda.synchronize()
    assert torch.equal(d[4][0], a[4][0]) and torch.equal(d[2][0], a[2][0]) and torch.equal(d[2][1], a[2][0])
    assert net.launch_count() > 0


# Inputs of 64 pixels or less per side leave P6 one pixel wide on that side; the second FPN downsample layer then runs a
# 3x3/s2/p1 conv whose odd phase is empty (its taps read only the zero padding).
SMALL_INPUT_CASES = [(c, H, W) for c in ("yolact_resnet50_config", "yolact_darknet53_config")
                     for H, W in ((64, 64), (550, 64))]


def _raw_heads(cfg_name, H, W, precision, seed=11):
    cfg = cfg_for(cfg_name)
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision=precision)
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 7))
    net.train()
    out = net(deterministic_input(1, H, W, seed=seed).cuda())
    return {k: out[k].cpu().numpy() for k in ("proto", "loc", "conf", "mask", "priors")}


@pytest.mark.parametrize("cfg_name,H,W", SMALL_INPUT_CASES, ids=lambda v: str(v))
def test_one_pixel_p6_tensor_cores_match_f32(cfg_name, H, W):
    ref = _raw_heads(cfg_name, H, W, "f32")
    got = _raw_heads(cfg_name, H, W, "f16x3")
    assert np.array_equal(got["priors"], ref["priors"])
    for k in ("proto", "loc", "conf", "mask"):
        assert np.isfinite(got[k]).all(), k
        e = rel_err(got[k], ref[k])
        print(cfg_name, H, W, k, "f16x3 vs f32 rel err %.2e" % e)
        assert e < RAW_TOL["f16x3"] + RAW_TOL["f32"], (k, e)


@pytest.mark.parametrize("cfg_name", ["yolact_resnet50_config", "yolact_darknet53_config"])
def test_one_pixel_p6_chain_identical_to_separate_launches(cfg_name, monkeypatch):
    monkeypatch.setenv("YB_SK", "0")
    heads = {}
    for chain in (0, 2):
        monkeypatch.setenv("YB_CHAIN", str(chain))
        heads[chain] = _raw_heads(cfg_name, 64, 64, "f16x3")
    for k in heads[0]:
        assert np.array_equal(heads[0][k], heads[2][k]), (k, float(np.abs(heads[0][k] - heads[2][k]).max()))
