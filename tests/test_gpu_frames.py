"""Yolact.infer_frames / forward_frames: uint8 BGR frames straight into the network, FastBaseTransform fused into the
tensor-core stem's loader (a separate kernel in the f32 mode).  The outputs must be bit-identical to the two-call path
infer_padded(FastBaseTransform(cfg)(frames)) on the same net, and match the CPU oracle at full size."""
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
from yolact_b200 import _lib
from yolact_b200.augmentations import FastBaseTransform

pytestmark = pytest.mark.gpu

SIZE = 152   # ResNet stem output 76x76 and Darknet's 152x152: neither a multiple of both 8 and 16
_nets = {}


def make_net(config, precision, size=SIZE):
    key = (config, precision, size)
    if key not in _nets:
        cfg = cfg_for(config)
        cfg.max_size = size
        yolact_b200.cfg.replace(cfg.copy())
        net = yolact_b200.Yolact(cfg, precision=precision)
        net.detect.use_fast_nms = True
        net.load_state_dict(deterministic_state_dict(net.state_dict(), 3))
        net.eval()
        _nets[key] = net
    net = _nets[key]
    yolact_b200.cfg.replace(net.cfg.copy())
    return net


def frames(B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, h, w, 3), generator=g, dtype=torch.uint8).cuda()


def two_call(net, f, cross_class):
    return net.infer_padded(FastBaseTransform(net.cfg)(f), cross_class=cross_class)


def assert_same(a, b, cross_class=False):
    """torch.equal on all six outputs.  cc_fast_nms writes only the first count rows of each image (rows past it keep
    whatever the buffer held, in infer_padded as well), so in that mode the row outputs are compared up to count."""
    assert torch.equal(a[4], b[4]), "counts differ"
    for i, (x, y) in enumerate(zip(a, b)):
        assert (x is None) == (y is None), i
        if x is None:
            continue
        if cross_class and i < 4:
            for img, n in enumerate(a[4].tolist()):
                assert torch.equal(x[img, :n], y[img, :n]), "output %d differs in image %d" % (i, img)
        else:
            assert torch.equal(x, y), "output %d differs" % i


# (B, h, w, preserve_aspect_ratio): downscaled, upscaled, not resized, and a non-square network input
FRAME_CASES = [(3, 200, 260, False), (1, 97, 130, False), (1, SIZE, SIZE, False), (3, 120, 200, True)]


@pytest.mark.parametrize("precision", ["f16x3", "f16tc", "f32"])
@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_darknet53_config"])
def test_infer_frames_is_bit_identical_to_fast_base_transform_then_infer_padded(config, precision):
    net = make_net(config, precision)
    for i, (B, h, w, par) in enumerate(FRAME_CASES):
        net.cfg.preserve_aspect_ratio = par
        try:
            f = frames(B, h, w, 10 + i)
            for cross_class in (False, True):
                ref = two_call(net, f, cross_class)
                got = net.infer_frames(f, cross_class=cross_class)
                torch.cuda.synchronize()
                assert_same(got, ref, cross_class)
        finally:
            net.cfg.preserve_aspect_ratio = False


@pytest.mark.parametrize("mode", ["subtract_means", "none"])
def test_infer_frames_other_transform_modes(mode):
    net = make_net("yolact_resnet50_config", "f16x3")
    net.cfg.normalize = False
    net.cfg.subtract_means = mode == "subtract_means"
    try:
        f = frames(2, 131, 170, 21)
        ref = two_call(net, f, False)
        got = net.infer_frames(f)
        torch.cuda.synchronize()
        assert_same(got, ref)
    finally:
        net.cfg.normalize, net.cfg.subtract_means = True, False


def test_graph_replay_and_isolation_between_frame_sizes_and_infer_padded():
    net = make_net("yolact_resnet50_config", "f16x3")
    fa, fb = frames(2, 180, 240, 31), frames(2, 100, 90, 32)
    a = [net.infer_frames(fa) for _ in range(3)]      # eager, capture, replay
    xa = FastBaseTransform(net.cfg)(fa)
    pa = [net.infer_padded(xa) for _ in range(3)]
    torch.cuda.synchronize()
    for r in a[1:] + pa:
        assert_same(r, a[0])
    b = [net.infer_frames(fb) for _ in range(3)]
    pa2 = net.infer_padded(xa)
    a2 = net.infer_frames(fa)
    b2 = net.infer_frames(fb)
    torch.cuda.synchronize()
    assert_same(a2, a[0])
    assert_same(pa2, a[0])
    assert_same(b2, b[0])
    assert not torch.equal(b[0][5], a[0][5])



def test_many_frame_sizes_share_one_input_and_repeat_their_results():
    """One network input size serves any number of frame sizes: cycling through six of them, then through them again,
    gives the same results both times and the same as the two-call path."""
    net = make_net("yolact_resnet50_config", "f16x3")
    fs = [frames(1, 100 + 7 * i, 140 + 5 * i, 60 + i) for i in range(6)]
    first = [net.infer_frames(f) for f in fs]
    again = [net.infer_frames(f) for f in fs]
    refs = [two_call(net, f, False) for f in fs]
    torch.cuda.synchronize()
    for a, b, r in zip(first, again, refs):
        assert_same(b, a)
        assert_same(b, r)

@pytest.mark.parametrize("precision,extra", [("f16x3", 0), ("f16tc", 0), ("f32", 1)])
def test_fused_path_launch_count(precision, extra):
    """On graph replay the half modes launch exactly what infer_padded does (the stem is replaced, nothing added); the
    f32 mode adds the one fast_base_transform kernel."""
    net = make_net("yolact_resnet50_config", precision)
    f = frames(1, 120, 160, 41)
    x = FastBaseTransform(net.cfg)(f)
    for _ in range(3):   # eager, capture, replay
        net.infer_frames(f)
        net.infer_padded(x)
    torch.cuda.synchronize()
    n0 = net.launch_count()
    net.infer_padded(x)
    n1 = net.launch_count()
    net.infer_frames(f)
    n2 = net.launch_count()
    torch.cuda.synchronize()
    assert n2 - n1 == (n1 - n0) + extra, (n1 - n0, n2 - n1)


def test_forward_frames_full_size_against_the_oracle():
    """One 480x640 frame through yolact_base at 550 (f16x3): forward_frames + postprocess's inputs against the CPU
    oracle's FastBaseTransform -> conv stack -> Detect."""
    cfg = cfg_for("yolact_base_config")
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    sd = deterministic_state_dict(net.state_dict(), 0)
    net.load_state_dict(sd)
    net.eval()
    img = np.random.RandomState(5).randint(0, 256, (1, 480, 640, 3)).astype(np.uint8)
    preds = net.forward_frames(torch.from_numpy(img).cuda())
    assert (yolact_b200.cfg._tmp_img_h, yolact_b200.cfg._tmp_img_w) == (550, 550)
    assert len(preds) == 1 and preds[0]["net"] is net
    det = preds[0]["detection"]
    x = torch.from_numpy(E.fast_base_transform(img, 550, 550, "normalize"))
    raw = O.ConvStackOracle(cfg, sd).forward(x)
    with torch.no_grad():
        ref = T.detect_one(raw["loc"][0], torch.softmax(raw["conf"], -1)[0], raw["mask"][0], raw["priors"],
                           cfg.nms_conf_thresh, cfg.nms_thresh, cfg.nms_top_k, cfg.max_num_detections)
    assert (det is None) == (ref is None)
    if ref is None:
        return
    got = {k: det[k].cpu().numpy() for k in ("class", "score", "box")}
    want = {k: ref[k].numpy() for k in ("class", "score", "box")}
    perm, ok = align(got, want)
    assert ok and (perm >= 0).all(), "class ids differ from the oracle beyond score ties"
    np.testing.assert_allclose(got["score"][perm], want["score"], atol=1e-3)
    np.testing.assert_allclose(got["box"][perm], want["box"], atol=1e-3)


def test_frame_input_errors():
    net = make_net("yolact_resnet50_config", "f16x3")
    f = frames(1, 64, 64, 51)
    with pytest.raises(_lib.YbError):
        net.infer_frames(f.cpu())
    with pytest.raises(ValueError, match="FastBaseTransform"):
        net.infer_frames(f.float())
    with pytest.raises(ValueError):
        net.infer_frames(f[..., :2].contiguous())
    with pytest.raises(ValueError):
        net.infer_frames(f[0])
    net.cfg.channel_order = "BGR"
    try:
        with pytest.raises(NotImplementedError):
            net.infer_frames(f)
    finally:
        net.cfg.channel_order = "RGB"
    net.train()
    try:
        with pytest.raises(RuntimeError):
            net.forward_frames(f)
    finally:
        net.eval()
