"""postprocess_list: every image of a list of detections postprocessed at its own size in one call (one launch per
kernel for the whole list).  Element i must equal postprocess(det_output, w_i, h_i, i, ...) bit for bit -- classes,
scores, boxes and masks, dtype and shape included -- and det_output must end as those calls leave it."""
import ctypes

import numpy as np
import pytest
import torch

import yolact_b200
from oracle.weights import deterministic_state_dict
from tests.helpers import cfg_for
from tests.test_gpu_frame_list import MIXED, frame
from tests.test_gpu_frames import SIZE, make_net
from yolact_b200 import _lib, output_utils
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.output_utils import postprocess, postprocess_list

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1   # include/yolact_b200.h

# MIXED plus a tiny image, an odd width that is neither a multiple of 4 nor of 32, and a 1080p frame
SIZES = MIXED + [(5, 7), (77, 101), (1080, 1920)]


def clone(preds):
    return [{"detection": None if p["detection"] is None else {k: v.clone() for k, v in p["detection"].items()},
             "net": p["net"]} for p in preds]


def per_image(preds, sizes, **kw):
    return [postprocess(preds, w, h, i, **kw) for i, (h, w) in enumerate(sizes)]


def assert_same_result(got, ref):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert len(g) == 4, i
        for j, (a, b) in enumerate(zip(g, r)):
            if isinstance(b, list):   # YOLACT++ [scores, scores * maskiou]
                assert isinstance(a, list) and len(a) == len(b), (i, j)
                for x, y in zip(a, b):
                    assert x.dtype == y.dtype and torch.equal(x, y), (i, j)
                continue
            assert a.dtype == b.dtype and a.shape == b.shape, (i, j, a.dtype, b.dtype, a.shape, b.shape)
            assert a.device == b.device and torch.equal(a, b), "image %d, output %d differs" % (i, j)


def assert_same_state(a, b):
    for i, (p, q) in enumerate(zip(a, b)):
        assert (p["detection"] is None) == (q["detection"] is None), i
        if p["detection"] is None:
            continue
        assert sorted(p["detection"]) == sorted(q["detection"]), i
        for k in p["detection"]:
            assert torch.equal(p["detection"][k], q["detection"][k]), (i, k)


def check(preds, sizes, **kw):
    """postprocess_list on preds against postprocess per image on an independent copy (the threshold filters dets in
    place); returns the list result."""
    ref_preds = clone(preds)
    ref = per_image(ref_preds, sizes, **kw)
    got = postprocess_list(preds, sizes, **kw)
    torch.cuda.synchronize()
    assert_same_result(got, ref)
    assert_same_state(preds, ref_preds)
    return got


def thresholds(preds):
    """0, one that cuts rows in some images (the median score of all rows) and one above every score of one image."""
    scores = [p["detection"]["score"] for p in preds if p["detection"] is not None]
    allsc = torch.cat(scores)
    return [0, float(allsc.median()), float(min(s.max() for s in scores))]


@pytest.fixture(scope="module")
def list_preds():
    net = make_net("yolact_resnet50_config", "f16x3")
    fs = [frame(h, w, 300 + i) for i, (h, w) in enumerate(SIZES)]
    preds = net.forward_frames(fs)
    assert sum(p["detection"] is not None for p in preds) >= 6
    return net, preds


@pytest.mark.parametrize("mask_format", ["f32", "u8", "bits"])
@pytest.mark.parametrize("crop_masks", [True, False])
@pytest.mark.parametrize("which_threshold", [0, 1, 2])
def test_list_is_bit_identical_to_postprocess_per_image(list_preds, mask_format, crop_masks, which_threshold):
    net, preds = list_preds
    make_net("yolact_resnet50_config", "f16x3")
    preds = clone(preds)
    thr = thresholds(preds)[which_threshold]
    got = check(preds, SIZES, mask_format=mask_format, crop_masks=crop_masks, score_threshold=thr)
    if which_threshold == 0:
        assert all(g[3].numel() > 0 for g, p in zip(got, preds) if p["detection"] is not None)
    if which_threshold == 2:
        assert any(g[3].numel() == 0 and p["detection"] is not None for g, p in zip(got, preds))


def test_none_detections_and_uniform_net_input(list_preds):
    net, preds = list_preds
    make_net("yolact_resnet50_config", "f16x3")
    preds = clone(preds)
    preds.insert(2, {"detection": None, "net": net})
    sizes = SIZES[:2] + [(40, 60)] + SIZES[2:]
    got = check(preds, sizes)
    assert all(t.numel() == 0 for t in got[2])
    # preds of net(x) at one input size, postprocessed at several sizes
    fs = torch.stack([frame(180, 240, 330 + i) for i in range(4)])
    preds = net(FastBaseTransform(net.cfg)(fs))
    check(preds, [(180, 240), (97, 33), (480, 640), (181, 241)], mask_format="bits")


@pytest.mark.parametrize("nms", ["cross_class", "traditional"])
def test_other_nms_modes(nms):
    net = make_net("yolact_resnet50_config", "f16x3")
    fs = [frame(h, w, 340 + i) for i, (h, w) in enumerate(MIXED)]
    try:
        if nms == "cross_class":
            net.detect.use_cross_class_nms = True
        else:
            net.detect.use_fast_nms = False
        preds = net.forward_frames(fs)
    finally:
        net.detect.use_cross_class_nms, net.detect.use_fast_nms = False, True
    for fmt in ("f32", "bits"):
        check(clone(preds), MIXED, mask_format=fmt)
    check(preds, MIXED, score_threshold=thresholds(preds)[1])


def test_full_size_yolact_base():
    """yolact_base at 550 on 480x640, 427x640 and 640x480 frames: the per-image path is checked against the oracle
    elsewhere, identity carries that over."""
    cfg = cfg_for("yolact_base_config")
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    rs = np.random.RandomState(7)
    sizes = [(480, 640), (427, 640), (640, 480)]
    preds = net.forward_frames([torch.from_numpy(rs.randint(0, 256, (h, w, 3)).astype(np.uint8)).cuda()
                                for h, w in sizes])
    assert all(p["detection"] is not None for p in preds)
    for fmt in ("f32", "bits"):
        check(clone(preds), sizes, mask_format=fmt)


def test_yolact_plus_maskiou_rescoring():
    net = make_net("yolact_plus_resnet50_config", "f16x3", 256)
    assert net.cfg.use_maskiou
    preds = net.forward_frames([frame(h, w, 350 + i) for i, (h, w) in enumerate(MIXED)])
    for fmt in ("f32", "bits"):
        got = check(clone(preds), MIXED, mask_format=fmt)
        assert any(isinstance(g[1], list) for g in got) == bool(getattr(net.cfg, "rescore_mask", False))
    check(clone(preds), MIXED, score_threshold=thresholds(preds)[1])
    save = yolact_b200.cfg.rescore_bbox
    yolact_b200.cfg.rescore_bbox = True
    try:
        got = check(clone(preds), MIXED)
        assert not any(isinstance(g[1], list) for g in got)
    finally:
        yolact_b200.cfg.rescore_bbox = save
    save = yolact_b200.cfg.eval_mask_branch
    yolact_b200.cfg.eval_mask_branch = False
    try:
        got = check(clone(preds), MIXED)
        for g, p in zip(got, preds):   # boxes only: the masks are the raw coefficients
            if p["detection"] is not None:
                assert torch.equal(g[3], p["detection"]["mask"])
    finally:
        yolact_b200.cfg.eval_mask_branch = save


@pytest.mark.parametrize("config,size,launches", [("yolact_resnet50_config", SIZE, 2),
                                                   ("yolact_plus_resnet50_config", 256, 10)])
def test_launches_do_not_grow_with_the_list_and_no_host_sync(config, size, launches):
    net = make_net(config, "f16x3", size)
    for B in (1, 3, 6):
        sizes = [(120 + 17 * i, 200 - 11 * i) for i in range(B)]
        preds = net.forward_frames([frame(h, w, 360 + i) for i, (h, w) in enumerate(sizes)])
        assert all(p["detection"] is not None for p in preds)
        postprocess_list(clone(preds), sizes)   # creates the ops handle and sizes the item table
        torch.cuda.synchronize()
        n0 = output_utils.launch_count() + net.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = postprocess_list(preds, sizes)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        n1 = output_utils.launch_count() + net.launch_count()
        assert n1 - n0 == launches, (B, n1 - n0)
        torch.cuda.synchronize()
        assert_same_result(got, per_image(preds, sizes))


def test_two_streams_share_the_item_table_in_order(list_preds):
    net, preds = list_preds
    make_net("yolact_resnet50_config", "f16x3")
    a, sa = clone(preds), SIZES
    b, sb = clone(preds[::-1]), [(h + 13, w + 5) for h, w in SIZES[::-1]]
    ref_a, ref_b = per_image(clone(a), sa, mask_format="bits"), per_image(clone(b), sb, mask_format="bits")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        got_a = postprocess_list(a, sa, mask_format="bits")
    with torch.cuda.stream(s2):
        got_b = postprocess_list(b, sb, mask_format="bits")
    torch.cuda.synchronize()
    assert_same_result(got_a, ref_a)
    assert_same_result(got_b, ref_b)


def test_python_errors(list_preds):
    net, preds = list_preds
    make_net("yolact_resnet50_config", "f16x3")
    with pytest.raises(ValueError):
        postprocess_list(clone(preds), SIZES[:-1])
    with pytest.raises(ValueError):
        postprocess_list(clone(preds), SIZES[:-1] + [(0, 10)])
    with pytest.raises(ValueError):
        postprocess_list(clone(preds), SIZES[:-1] + [(10, -1)])
    bad = clone(preds)
    live = [p for p in bad if p["detection"] is not None]
    live[-1]["detection"]["proto"] = live[-1]["detection"]["proto"][:-1].contiguous()
    with pytest.raises(ValueError, match="proto"):
        postprocess_list(bad, SIZES)
    cpu = clone(preds)
    for p in cpu:
        if p["detection"] is not None:
            p["detection"] = {k: v.cpu() for k, v in p["detection"].items()}
    with pytest.raises(_lib.YbError):
        postprocess_list(cpu, SIZES)
    with pytest.raises(NotImplementedError):
        postprocess_list(clone(preds), SIZES, interpolation_mode="nearest")
    with pytest.raises(NotImplementedError):
        postprocess_list(clone(preds), SIZES, visualize_lincomb=True)
    # kept rows that are not the leading rows: refused, and nothing is filtered
    rev = clone(preds)
    d = next(p["detection"] for p in rev if p["detection"] is not None and p["detection"]["score"].numel() > 2)
    for k in list(d):
        if k != "proto":
            d[k] = d[k].flip(0)
    before = clone(rev)
    thr = float(d["score"].median())
    with pytest.raises(ValueError, match="leading rows"):
        postprocess_list(rev, SIZES, score_threshold=thr)
    assert_same_state(rev, before)


def test_c_abi_rejects_bad_items():
    """Null inputs with n > 0, negative n, non-positive sizes, misaligned masks and host memory are refused before
    anything runs; the handle keeps working."""
    make_net("yolact_resnet50_config", "f16x3")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = output_utils._ops_handle(dev, 32)
    st = _lib.current_stream(dev)
    g = torch.Generator(device="cuda").manual_seed(5)
    proto = torch.rand(20, 24, 32, device=dev, generator=g)
    coef = torch.randn(3, 32, device=dev, generator=g)
    box = torch.tensor([[0.1, 0.2, 0.6, 0.7], [0.0, 0.0, 1.0, 1.0], [0.3, 0.3, 0.4, 0.9]], device=dev)
    masks = torch.empty(3 * 40 * 50 + 8, device=dev)
    boxes_px = torch.empty(3, 4, dtype=torch.int64, device=dev)
    host = np.zeros((3, 4), np.float32)

    def call(**kw):
        f = dict(proto=proto.data_ptr(), coef=coef.data_ptr(), box=box.data_ptr(), masks=masks.data_ptr(),
                 boxes_px=boxes_px.data_ptr(), proto_masks=None, n=3, out_h=40, out_w=50)
        f.update(kw)
        items = (_lib.YbPostItem * 2)(_lib.YbPostItem(**f), _lib.YbPostItem(**dict(f, n=0)))
        return lib.yb_postprocess_list(h, items, 2, 20, 24, 32, 1, _lib.YB_MASK_F32, st)

    assert call() == 0, lib.yb_last_error()
    torch.cuda.synchronize()
    want_masks, want_px, _ = output_utils.assemble_masks(proto, coef, box, 40, 50)
    torch.cuda.synchronize()
    assert torch.equal(masks[:3 * 40 * 50].view(3, 40, 50), want_masks) and torch.equal(boxes_px, want_px)
    for bad in (dict(proto=None), dict(coef=None), dict(box=None), dict(n=-1), dict(out_h=0), dict(out_w=-2),
                dict(masks=masks.data_ptr() + 4), dict(box=host.ctypes.data), dict(boxes_px=host.ctypes.data)):
        assert call(**bad) == YB_ERR_INVALID, bad
    assert call(proto=None, coef=None, box=None, n=0) == 0   # n == 0 needs no inputs
    torch.cuda.synchronize()
    masks.zero_()
    assert call() == 0, lib.yb_last_error()   # the handle still works
    torch.cuda.synchronize()
    assert torch.equal(masks[:3 * 40 * 50].view(3, 40, 50), want_masks)
