"""render_masks: prep_display's GPU part for a list of frames, straight from the detections.  Every image and every drawn
row must equal today's composition -- postprocess(mask_format='u8') with rescore_bbox, a stable descending sort, the
top_k rows, the score cut, the palette and display_blend -- bit for bit, and the reference's own prep_display output
within the blend's known +-1 truncation."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import yolact_b200
from oracle.weights import deterministic_state_dict
from tests.conftest import load_golden
from tests.helpers import cfg_for
from yolact_b200 import _lib
from yolact_b200 import config as ybcfg
from yolact_b200.display import _palette, render_masks
from yolact_b200.eval_utils import display_blend, get_color
from yolact_b200.output_utils import _ops_handle, launch_count, postprocess

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1   # include/yolact_b200.h
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_dets(n, ph, pw, seed, score_lo=0.05, ties=False):
    r = np.random.RandomState(seed)
    proto = np.maximum(r.standard_normal((ph, pw, 32)), 0).astype(np.float32)
    coef = np.tanh(r.standard_normal((n, 32)) * 1.5).astype(np.float32)
    c = r.uniform(0.05, 0.95, (n, 2))
    wh = r.uniform(0.05, 0.7, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(np.float32)
    if ties:
        score = r.choice(np.float32([0.9, 0.6, 0.4, 0.2]), n).astype(np.float32)
    else:
        score = (score_lo + (0.95 - score_lo) * r.permutation(n) / max(n, 1)).astype(np.float32)   # distinct
    cls = r.randint(0, 80, n).astype(np.int64)
    return {"box": cuda(box), "mask": cuda(coef), "class": cuda(cls), "score": cuda(score), "proto": cuda(proto)}


def composition(det, frame, top_k, score_threshold, class_color=False, crop_masks=True, mask_alpha=0.45, net=None):
    """A caller's prep_display today (tests/test_gpu_eval_rows.py::_caller_prep_display) with a stable sort, and the
    drawn rows it would hand to OpenCV."""
    dets = [{"detection": dict(det) if det is not None else None, "net": net}]   # postprocess filters in place
    cfg = ybcfg.cfg
    save, cfg.rescore_bbox = cfg.rescore_bbox, True
    try:
        t = postprocess(dets, int(frame.shape[1]), int(frame.shape[0]), crop_masks=crop_masks,
                        score_threshold=score_threshold, mask_format="u8")
    finally:
        cfg.rescore_bbox = save
    if t[1].numel() == 0:
        n, classes, scores, boxes, masks = 0, np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros((0, 4)), None
    else:
        idx = torch.sort(t[1], descending=True, stable=True)[1][:top_k]
        masks = t[3][idx]
        classes, scores, boxes = t[0][idx].cpu().numpy(), t[1][idx].cpu().numpy(), t[2][idx].cpu().numpy()
        n = min(top_k, classes.shape[0])
        for j in range(n):
            if scores[j] < score_threshold:
                n = j
                break
    colors = [[c / 255.0 for c in get_color(j, classes, class_color, bgr=True)] for j in range(n)]
    img = display_blend(frame.float(), masks[:n] if n else None, colors if n else None, mask_alpha).cpu().numpy()
    return img, n, classes[:n], scores[:n], boxes[:n]


def check(dets, frames, top_k, thr, net=None, **kw):
    det_output = [{"detection": d, "net": net} for d in dets]
    images, drawn = render_masks(det_output, frames, top_k=top_k, score_threshold=thr, **kw)
    num = drawn["num"].cpu().numpy()
    for i, (d, f) in enumerate(zip(dets, frames)):
        img, n, classes, scores, boxes = composition(d, f, top_k, thr, net=net, **kw)
        assert images[i].dtype == torch.uint8 and tuple(images[i].shape) == tuple(f.shape)
        assert np.array_equal(images[i].cpu().numpy(), img), (i, tuple(f.shape), top_k, thr, kw)
        assert num[i] == n, (i, num[i], n)
        assert np.array_equal(drawn["classes"][i, :n].cpu().numpy(), classes)
        assert np.array_equal(drawn["scores"][i, :n].cpu().numpy(), scores)
        assert np.array_equal(drawn["boxes"][i, :n].cpu().numpy(), boxes)
        assert not drawn["classes"][i, n:].any() and not drawn["boxes"][i, n:].any()
    return images, drawn


SIZES = [(5, 7), (77, 101), (203, 277), (550, 550), (480, 640), (1080, 1920)]


def frames_for(sizes, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    fs = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for h, w in sizes]
    return fs if dtype == torch.uint8 else [f.float() for f in fs]


@pytest.mark.parametrize("top_k", [1, 5, 15, 100])
@pytest.mark.parametrize("thr", [0, 0.15, 0.3])
def test_render_matches_the_composition(top_k, thr):
    ybcfg.set_cfg("yolact_base_config")
    ns = [37, 0, 100, 1, 64, 99]   # odd n, n = 0, and every size in one list
    dets = [make_dets(n, 138, 138, 100 + i) if n else None for i, n in enumerate(ns)]
    dets[3] = make_dets(9, 138, 138, 7, score_lo=0.0)
    dets[3]["score"] = dets[3]["score"] * 0.1   # every row below the thresholds
    for crop in (True, False):
        for class_color in (False, True):
            check(dets, frames_for(SIZES, top_k, torch.uint8), top_k, thr, crop_masks=crop, class_color=class_color)
    check(dets, frames_for(SIZES, 1 + top_k, torch.float32), top_k, thr)


def test_render_im700_prototypes_and_a_batch_tensor():
    ybcfg.set_cfg("yolact_im700_config")
    dets = [make_dets(n, 176, 176, 300 + n) for n in (100, 31)]
    check(dets, frames_for([(700, 700), (480, 640)], 5, torch.uint8), 15, 0.15)
    batch = torch.stack(frames_for([(120, 90)] * 3, 6, torch.uint8))
    dets3 = [make_dets(n, 176, 176, 310 + n) for n in (3, 50, 11)]
    images, _ = render_masks([{"detection": d, "net": None} for d in dets3], batch, top_k=5)
    alone = [render_masks([{"detection": d, "net": None}], [f], top_k=5)[0][0] for d, f in zip(dets3, batch)]
    assert all(torch.equal(a, b) for a, b in zip(images, alone))
    ybcfg.set_cfg("yolact_base_config")


def test_ties_keep_the_lower_row_first():
    ybcfg.set_cfg("yolact_base_config")
    d = make_dets(40, 138, 138, 11, ties=True)
    frames = frames_for([(203, 277)], 12, torch.uint8)
    _, drawn = check([d], frames, 15, 0)
    order = np.argsort(-d["score"].cpu().numpy(), kind="stable")[:15]
    assert np.array_equal(drawn["classes"][0].cpu().numpy(), d["class"].cpu().numpy()[order])


def _golden_dets():
    g = load_golden("eval_unit")
    det = {"box": cuda(g["disp_box"]), "mask": cuda(g["disp_coef"]), "class": cuda(g["disp_cls"]),
           "score": cuda(g["disp_score"]), "proto": cuda(g["disp_proto"])}
    return g, det, cuda(g["disp_frame"])


@pytest.mark.parametrize("tag,kw", [("masks", dict(top_k=8, score_threshold=0.15)),
                                    ("classcolor", dict(top_k=15, score_threshold=0.3, class_color=True))])
def test_render_matches_the_reference_prep_display(tag, kw):
    ybcfg.set_cfg("yolact_base_config")
    g, det, frame = _golden_dets()
    for f in (frame, frame.float()):
        images, _ = render_masks([{"detection": det, "net": None}], [f], **kw)
        out, ref = images[0].cpu().numpy(), g["disp_" + tag]
        diff = np.abs(out.astype(np.int32) - ref.astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 2e-3                  # .byte() truncation: +-1 LSB, rarely


COCO_CLASSES = ('person', 'bicycle', 'car', 'motorcycle', 'airplane', 'bus', 'train', 'truck', 'boat', 'traffic light',
                'fire hydrant', 'stop sign', 'parking meter', 'bench', 'bird', 'cat', 'dog', 'horse', 'sheep', 'cow',
                'elephant', 'bear', 'zebra', 'giraffe', 'backpack', 'umbrella', 'handbag', 'tie', 'suitcase', 'frisbee',
                'skis', 'snowboard', 'sports ball', 'kite', 'baseball bat', 'baseball glove', 'skateboard', 'surfboard',
                'tennis racket', 'bottle', 'wine glass', 'cup', 'fork', 'knife', 'spoon', 'bowl', 'banana', 'apple',
                'sandwich', 'orange', 'broccoli', 'carrot', 'hot dog', 'pizza', 'donut', 'cake', 'chair', 'couch',
                'potted plant', 'bed', 'dining table', 'toilet', 'tv', 'laptop', 'mouse', 'remote', 'keyboard',
                'cell phone', 'microwave', 'oven', 'toaster', 'sink', 'refrigerator', 'book', 'clock', 'vase',
                'scissors', 'teddy bear', 'hair drier', 'toothbrush')


def test_render_then_opencv_text_matches_the_reference_full_display():
    """eval.py's default display (top_k 5, score_threshold 0.15, text and boxes on): the boxes and text are drawn by the
    caller from `drawn` with one device-to-host copy, as eval.py:236-259 does."""
    cv2 = pytest.importorskip("cv2")
    ybcfg.set_cfg("yolact_base_config")
    g, det, frame = _golden_dets()
    images, drawn = render_masks([{"detection": det, "net": None}], [frame], top_k=5, score_threshold=0.15)
    img = images[0].cpu().numpy()
    num, classes, scores, boxes = (drawn[k][0].cpu().numpy() for k in ("num", "classes", "scores", "boxes"))
    for j in reversed(range(int(num))):
        x1, y1, x2, y2 = (int(v) for v in boxes[j])
        color = get_color(j, classes, False, bgr=True)
        cv2.rectangle(img, (x1, y1), (x2, y2), color, 1)
        text_str = '%s: %.2f' % (COCO_CLASSES[classes[j]], scores[j])
        text_w, text_h = cv2.getTextSize(text_str, cv2.FONT_HERSHEY_DUPLEX, 0.6, 1)[0]
        cv2.rectangle(img, (x1, y1), (x1 + text_w, y1 - text_h - 4), color, -1)
        cv2.putText(img, text_str, (x1, y1 - 3), cv2.FONT_HERSHEY_DUPLEX, 0.6, [255, 255, 255], 1, cv2.LINE_AA)
    diff = np.abs(img.astype(np.int32) - g["disp_full"].astype(np.int32))
    assert (diff > 1).mean() < 2e-3 and (diff > 0).mean() < 2e-3


def _net(config):
    cfg = cfg_for(config)
    cfg.max_size = 256 if cfg.use_maskiou else 160   # FastMaskIoUNet's five stride-2 convs need 64x64 prototypes
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 5))
    net.eval()
    return net


@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_plus_resnet50_config"])
def test_through_the_network(config):
    net = _net(config)
    g = torch.Generator().manual_seed(17)
    sizes = [(200, 260), (97, 130), (151, 77), (256, 256), (63, 301)]
    fs = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for h, w in sizes]
    preds = net.forward_frames(fs)
    assert any(p["detection"] is not None for p in preds)
    for thr in (0, 0.15):
        images, drawn = render_masks(preds, fs, top_k=15, score_threshold=thr)
        for i, f in enumerate(fs):
            one, d1 = render_masks(preds[i:i + 1], [f], top_k=15, score_threshold=thr)
            assert torch.equal(one[0], images[i])
            assert all(torch.equal(d1[k][0], drawn[k][i]) for k in drawn)
            img, n, classes, scores, boxes = composition(preds[i]["detection"], f, 15, thr, net=net)
            assert np.array_equal(images[i].cpu().numpy(), img), (config, thr, i)
            assert int(drawn["num"][i]) == n and np.array_equal(drawn["scores"][i, :n].cpu().numpy(), scores)
    # launches do not grow with the list, and the call never syncs the host
    torch.cuda.synchronize()
    counts = []
    for k in (1, 5):
        n0 = launch_count()
        render_masks(preds[:k], fs[:k], top_k=15, score_threshold=0.15)
        counts.append(launch_count() - n0)
    assert counts[0] == counts[1], counts
    torch.cuda.set_sync_debug_mode("error")
    try:
        render_masks(preds, fs, top_k=15, score_threshold=0.3)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_large_frames_in_a_fresh_process():
    """2160x3840 with top_k 100, and a frame smaller than the prototypes with top_k 100, whose sigmoid groups need more
    than 48 KB of shared memory: the opt-in runs in a process that has not launched the kernel before."""
    code = r'''
import sys, torch
sys.path.insert(0, %r)
from tests.test_gpu_render import make_dets, frames_for, check
from yolact_b200 import config as ybcfg
ybcfg.set_cfg("yolact_base_config")
dets = [make_dets(100, 138, 138, 900), make_dets(100, 138, 138, 901)]
check(dets, frames_for([(2160, 3840), (40, 30)], 3, torch.uint8), 100, 0)
print("ok")
''' % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_c_abi_rejects_bad_items():
    ybcfg.set_cfg("yolact_base_config")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = _ops_handle(dev, 32)
    d = make_dets(6, 138, 138, 40)
    frame = frames_for([(20, 30)], 41, torch.uint8)[0]
    out = torch.empty_like(frame)
    host = np.zeros((20, 30, 3), np.uint8)
    pal = _palette(dev)

    def item(**over):
        it = _lib.YbRenderItem(frame.data_ptr(), out.data_ptr(), d["proto"].data_ptr(), d["mask"].data_ptr(),
                               d["box"].data_ptr(), d["class"].data_ptr(), d["score"].data_ptr(), d["score"].data_ptr(),
                               None, None, None, None, 6, 20, 30)
        for k, v in over.items():
            setattr(it, k, v)
        return it

    def call(it, top_k=5, P=len(ybcfg.COLORS)):
        items = (_lib.YbRenderItem * 1)(it)
        return lib.yb_render_list(h, items, 1, 1, 138, 138, 32, 1, top_k, 0.0, 0, 0.45, _lib.ptr(pal), P,
                                  _lib.current_stream(dev))

    assert call(item()) == 0, lib.yb_last_error()
    for bad in (dict(frame=None), dict(out=None), dict(h=0), dict(w=-2), dict(n=-1), dict(cls=None),
                dict(det_score=None), dict(frame=host.ctypes.data)):
        assert call(item(**bad)) == YB_ERR_INVALID, bad
        assert lib.yb_last_error()
    assert call(item(), top_k=0) == YB_ERR_INVALID
    assert call(item(), P=0) == YB_ERR_INVALID
    assert call(item(frame=host.ctypes.data)) == YB_ERR_INVALID and b"device memory" in lib.yb_last_error()
    torch.cuda.synchronize()
    assert call(item(n=0, proto=None, coef=None)) == 0   # the handle is still usable
