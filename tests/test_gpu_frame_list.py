"""Yolact.infer_frames / forward_frames on a list of differently sized uint8 BGR frames: one call, one graph per
transform and NMS mode whatever the sizes.  The outputs must be bit-identical to the two-call path
infer_padded(torch.cat([FastBaseTransform(cfg)(f[None]) for f in frames])) on the same net, and match the CPU oracle at
full size."""
import ctypes

import numpy as np
import pytest
import torch

import yolact_b200
from oracle import eval_oracle as E
from oracle import torch_port as T
from oracle import yolact_oracle as O
from oracle.weights import deterministic_state_dict
from tests.helpers import cfg_for
from tests.parity_utils import align
from tests.test_gpu_frames import SIZE, assert_same, make_net
from yolact_b200 import _lib
from yolact_b200.augmentations import FastBaseTransform
from yolact_b200.output_utils import postprocess

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1   # include/yolact_b200.h


def frame(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda()


def two_call(net, fs, cross_class=None):
    x = torch.cat([FastBaseTransform(net.cfg)(f[None]) for f in fs])
    return net.infer_padded(x, cross_class=cross_class)


# downscaled, upscaled, odd-sized (both ways) and exactly the network input size, in one list
MIXED = [(200, 260), (97, 130), (151, 77), (SIZE, SIZE), (63, 301)]


@pytest.mark.parametrize("precision", ["f16x3", "f16tc", "f32"])
@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_darknet53_config"])
def test_frame_list_is_bit_identical_to_fast_base_transform_then_infer_padded(config, precision):
    net = make_net(config, precision)
    fs = [frame(h, w, 100 + i) for i, (h, w) in enumerate(MIXED)]
    for cross_class in (False, True):
        ref = two_call(net, fs, cross_class)
        got = [net.infer_frames(fs, cross_class=cross_class) for _ in range(3)]   # eager, capture, replay
        torch.cuda.synchronize()
        for g in got:
            assert_same(g, ref, cross_class)


@pytest.mark.parametrize("mode", ["subtract_means", "none"])
def test_frame_list_other_transform_modes(mode):
    net = make_net("yolact_resnet50_config", "f16x3")
    net.cfg.normalize = False
    net.cfg.subtract_means = mode == "subtract_means"
    try:
        fs = [frame(h, w, 120 + i) for i, (h, w) in enumerate(MIXED[:3])]
        ref = two_call(net, fs)
        got = net.infer_frames(tuple(fs))
        torch.cuda.synchronize()
        assert_same(got, ref)
    finally:
        net.cfg.normalize, net.cfg.subtract_means = True, False


def test_a_list_of_same_size_frames_matches_the_stacked_tensor():
    net = make_net("yolact_resnet50_config", "f16x3")
    fs = [frame(180, 240, 130 + i) for i in range(3)]
    ref = net.infer_frames(torch.stack(fs))
    got = net.infer_frames(fs)
    torch.cuda.synchronize()
    assert_same(got, ref)


@pytest.mark.parametrize("precision,extra", [("f16x3", 0), ("f16tc", 0), ("f32", 1)])
def test_frame_sizes_leave_no_state_and_replay_one_graph(precision, extra):
    """12 distinct sizes in three B=4 lists, then the lists again: every output is the two-call path's.  On replay a
    list call launches what infer_padded does (the half modes replace the stem; f32 adds its transform kernel), also
    for a list of sizes the executor has never seen."""
    net = make_net("yolact_resnet50_config", precision)
    sizes = [(90 + 11 * i, 170 - 7 * i) for i in range(12)]
    lists = [[frame(h, w, 140 + 4 * j + i) for i, (h, w) in enumerate(sizes[4 * j:4 * j + 4])] for j in range(3)]
    refs = [two_call(net, fs) for fs in lists]
    first = [net.infer_frames(fs) for fs in lists]
    again = [net.infer_frames(fs) for fs in lists]
    torch.cuda.synchronize()
    for a, b, r in zip(first, again, refs):
        assert_same(a, r)
        assert_same(b, r)
    x = torch.cat([FastBaseTransform(net.cfg)(f[None]) for f in lists[0]])
    for _ in range(3):
        net.infer_padded(x)
    unseen = [frame(h + 1, w + 3, 170 + i) for i, (h, w) in enumerate(sizes[:4])]
    torch.cuda.synchronize()
    n0 = net.launch_count()
    net.infer_padded(x)
    n1 = net.launch_count()
    net.infer_frames(lists[1])
    n2 = net.launch_count()
    got = net.infer_frames(unseen)
    n3 = net.launch_count()
    ref = two_call(net, unseen)
    torch.cuda.synchronize()
    assert n2 - n1 == (n1 - n0) + extra, (n1 - n0, n2 - n1)
    assert n3 - n2 == (n1 - n0) + extra, (n1 - n0, n3 - n2)
    assert_same(got, ref)


def test_interleaved_tensor_list_and_padded_calls_are_isolated():
    net = make_net("yolact_resnet50_config", "f16x3")
    ft = torch.stack([frame(120, 200, 180 + i) for i in range(len(MIXED))])
    fl = [frame(h, w, 190 + i) for i, (h, w) in enumerate(MIXED)]
    xp = FastBaseTransform(net.cfg)(torch.stack([frame(300, 150, 200 + i) for i in range(len(MIXED))]))
    alone = [net.infer_frames(ft), net.infer_frames(fl), net.infer_padded(xp)]
    for _ in range(3):
        got = [net.infer_frames(ft), net.infer_frames(fl), net.infer_padded(xp)]
        torch.cuda.synchronize()
        for g, a in zip(got, alone):
            assert_same(g, a)
    top_k = net.detect.top_k
    net.detect.top_k = 50   # yb_set_detect_params: drops every captured graph
    try:
        got, ref = net.infer_frames(fl), two_call(net, fl)
        again = net.infer_frames(fl)
        torch.cuda.synchronize()
        assert_same(got, ref)
        assert_same(again, ref)
    finally:
        net.detect.top_k = top_k
    got = net.infer_frames(fl)
    torch.cuda.synchronize()
    assert_same(got, alone[1])


def test_forward_frames_list_then_postprocess_at_each_image_size():
    net = make_net("yolact_resnet50_config", "f16x3")
    fs = [frame(h, w, 210 + i) for i, (h, w) in enumerate(MIXED)]
    ref_preds = net(torch.cat([FastBaseTransform(net.cfg)(f[None]) for f in fs]))
    ref = [postprocess(ref_preds, f.shape[1], f.shape[0], i) for i, f in enumerate(fs)]
    preds = net.forward_frames(fs)
    assert (yolact_b200.cfg._tmp_img_h, yolact_b200.cfg._tmp_img_w) == (SIZE, SIZE)
    assert len(preds) == len(fs) and all(p["net"] is net for p in preds)
    got = [postprocess(preds, f.shape[1], f.shape[0], i) for i, f in enumerate(fs)]
    torch.cuda.synchronize()
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g[3].shape[1:] == fs[i].shape[:2] or g[3].numel() == 0
        for a, b in zip(g, r):
            assert torch.equal(a, b), i


def test_forward_frames_list_full_size_against_the_oracle():
    """480x640, 427x640 and 640x480 frames in one list through yolact_base at 550 (f16x3): forward_frames' detections
    against the CPU oracle's FastBaseTransform -> conv stack -> Detect, image by image."""
    cfg = cfg_for("yolact_base_config")
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    sd = deterministic_state_dict(net.state_dict(), 0)
    net.load_state_dict(sd)
    net.eval()
    rs = np.random.RandomState(6)
    imgs = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in ((480, 640), (427, 640), (640, 480))]
    preds = net.forward_frames([torch.from_numpy(im).cuda() for im in imgs])
    assert len(preds) == 3
    oracle = O.ConvStackOracle(cfg, sd)
    for i, im in enumerate(imgs):
        det = preds[i]["detection"]
        x = torch.from_numpy(E.fast_base_transform(im[None], 550, 550, "normalize"))
        raw = oracle.forward(x)
        with torch.no_grad():
            ref = T.detect_one(raw["loc"][0], torch.softmax(raw["conf"], -1)[0], raw["mask"][0], raw["priors"],
                               cfg.nms_conf_thresh, cfg.nms_thresh, cfg.nms_top_k, cfg.max_num_detections)
        assert (det is None) == (ref is None), i
        if ref is None:
            continue
        got = {k: det[k].cpu().numpy() for k in ("class", "score", "box")}
        want = {k: ref[k].numpy() for k in ("class", "score", "box")}
        perm, ok = align(got, want)
        assert ok and (perm >= 0).all(), "image %d: class ids differ from the oracle beyond score ties" % i
        np.testing.assert_allclose(got["score"][perm], want["score"], atol=1e-3)
        np.testing.assert_allclose(got["box"][perm], want["box"], atol=1e-3)


def test_frame_list_errors():
    net = make_net("yolact_resnet50_config", "f16x3")
    f = frame(64, 64, 220)
    with pytest.raises(ValueError, match="empty"):
        net.infer_frames([])
    with pytest.raises(_lib.YbError):
        net.infer_frames([f, f.cpu()])
    with pytest.raises(ValueError, match="uint8"):
        net.infer_frames([f, f.float()])
    with pytest.raises(ValueError):
        net.infer_frames([f, f[..., :2].contiguous()])
    with pytest.raises(ValueError):
        net.infer_frames([f, f[None]])
    net.cfg.preserve_aspect_ratio = True
    try:
        with pytest.raises(ValueError, match="preserve_aspect_ratio"):
            net.infer_frames([frame(100, 200, 221), frame(200, 100, 222)])
    finally:
        net.cfg.preserve_aspect_ratio = False


def test_frame_list_c_abi_rejects_bad_frames():
    """Null frame pointers, non-positive sizes and host memory are refused before anything runs."""
    net = make_net("yolact_resnet50_config", "f16x3")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = net._handle_for(dev)
    mode, M, out = net._detect_outputs(h, dev, 2, SIZE, SIZE, None)
    f = frame(64, 80, 230)
    host = np.zeros((64, 80, 3), np.uint8)
    mean = (ctypes.c_float * 3)(*yolact_b200.config.MEANS)
    std = (ctypes.c_float * 3)(*yolact_b200.config.STD)

    def call(ptrs, hw):
        return lib.yb_infer_frame_list(h, (ctypes.c_void_p * 2)(*ptrs), (ctypes.c_int32 * 4)(*hw), 2, SIZE, SIZE,
                                       _lib.YB_XFORM_NORMALIZE, mean, std, mode, M, *[_lib.ptr(t) for t in out],
                                       _lib.current_stream(dev))

    good = [f.data_ptr(), f.data_ptr()]
    assert call(good, [64, 80, 64, 80]) == 0, _lib.load().yb_last_error()
    assert call([f.data_ptr(), None], [64, 80, 64, 80]) == YB_ERR_INVALID
    assert call(good, [64, 80, 0, 80]) == YB_ERR_INVALID
    assert call(good, [64, 80, 64, -3]) == YB_ERR_INVALID
    assert call([f.data_ptr(), host.ctypes.data], [64, 80, 64, 80]) == YB_ERR_INVALID
    torch.cuda.synchronize()
    assert net.infer_frames([f, f]) is not None   # the handle is still usable


def test_frames_c_abi_rejects_host_memory():
    """yb_infer_frames reads its batch in place: a host d_img is refused before anything runs."""
    net = make_net("yolact_resnet50_config", "f16x3")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = net._handle_for(dev)
    mode, M, out = net._detect_outputs(h, dev, 2, SIZE, SIZE, None)
    f = torch.stack([frame(64, 80, 231), frame(64, 80, 232)])
    host = np.zeros((2, 64, 80, 3), np.uint8)
    mean = (ctypes.c_float * 3)(*yolact_b200.config.MEANS)
    std = (ctypes.c_float * 3)(*yolact_b200.config.STD)

    def call(ptr):
        return lib.yb_infer_frames(h, ptr, 2, 64, 80, SIZE, SIZE, _lib.YB_XFORM_NORMALIZE, mean, std, mode, M,
                                   *[_lib.ptr(t) for t in out], _lib.current_stream(dev))

    assert call(f.data_ptr()) == 0, lib.yb_last_error()
    assert call(host.ctypes.data) == YB_ERR_INVALID
    torch.cuda.synchronize()
    assert net.infer_frames(f) is not None   # the handle is still usable
