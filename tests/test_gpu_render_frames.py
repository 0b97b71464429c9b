"""Yolact.render_frames (frames -> drawn frames with no host sync), the --display_fps box and --display_masks=False of
render_masks, yb_render_list_ex's refusals, and integration.use_b200.install_display against the reference's own
prep_display (tests/golden/display_unit.npz, scripts/gen_display_golden.py)."""
import os
import types

import numpy as np
import pytest
import torch

import yolact_b200
from tests.test_gpu_render import _net, frames_for, make_dets
from yolact_b200 import _lib
from yolact_b200 import config as ybcfg
from yolact_b200.display import _palette, render_masks
from yolact_b200.eval_utils import get_color
from yolact_b200.output_utils import _ops_handle, launch_count, postprocess

pytestmark = pytest.mark.gpu

YB_ERR_INVALID = -1   # include/yolact_b200.h
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "display_unit.npz")


def same(a, b):
    images_a, drawn_a = a
    images_b, drawn_b = b
    assert len(images_a) == len(images_b)
    for x, y in zip(images_a, images_b):
        assert torch.equal(x, y)
    for key in ("num", "classes", "scores", "boxes"):
        assert torch.equal(drawn_a[key], drawn_b[key]), key


_nets = {}


def net_for(config, precision):
    key = (config, precision)
    if key not in _nets:
        net = _net(config)
        if precision != "f16x3":
            cfg = net.cfg
            net = yolact_b200.Yolact(cfg, precision=precision)
            net.detect.use_fast_nms = True
            from oracle.weights import deterministic_state_dict
            net.load_state_dict(deterministic_state_dict(net.state_dict(), 5))
            net.eval()
        _nets[key] = net
    net = _nets[key]
    yolact_b200.cfg.replace(net.cfg.copy())
    return net


def mixed_frames(seed):
    g = torch.Generator().manual_seed(seed)
    sizes = [(200, 260), (9, 13), (151, 77), (256, 256), (63, 301)]   # (9, 13): smaller than the prototypes
    return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for h, w in sizes]


def batch_frames(seed, B=4, h=120, w=170):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, h, w, 3), generator=g, dtype=torch.uint8).cuda()


def check_against_list_path(net, frames, **kw):
    want = render_masks(net.forward_frames(frames), frames, **kw)
    got = net.render_frames(frames, **kw)
    same(got, want)
    return got


@pytest.mark.parametrize("precision", ["f16x3", "f32"])
@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_plus_resnet50_config", "yolact_darknet53_config"])
def test_render_frames_equals_forward_frames_then_render_masks(config, precision):
    net = net_for(config, precision)
    inputs = {"list": mixed_frames(31), "batch": batch_frames(32)}
    for name, frames in inputs.items():
        preds = net.forward_frames(frames)
        assert any(p["detection"] is not None for p in preds), (config, name)
        for top_k in (1, 5, 15, 100):
            for thr in (0, 0.15, 0.3):
                check_against_list_path(net, frames, top_k=top_k, score_threshold=thr)
        check_against_list_path(net, frames, top_k=15, class_color=True)
        check_against_list_path(net, frames, top_k=15, score_threshold=0.15, crop_masks=False)
        check_against_list_path(net, frames, top_k=5, fps_box=(107, 14), draw_masks=False)
        check_against_list_path(net, frames, top_k=5, score_threshold=0.15, fps_box=(300, 14), mask_alpha=0.3)
    # cfg.eval_mask_branch off (--detect): rows are selected, nothing is drawn
    yolact_b200.cfg.eval_mask_branch = False
    try:
        check_against_list_path(net, inputs["list"], top_k=15, score_threshold=0.15)
    finally:
        yolact_b200.cfg.eval_mask_branch = True


def test_images_without_detections():
    net = net_for("yolact_resnet50_config", "f16x3")
    frames = mixed_frames(41)
    saved = net.detect.conf_thresh
    net.detect.conf_thresh = 1.5   # no score passes: every image is empty
    try:
        preds = net.forward_frames(frames)
        assert all(p["detection"] is None for p in preds)
        images, drawn = check_against_list_path(net, frames, top_k=5, fps_box=(20, 3))
        assert not drawn["num"].any()
    finally:
        net.detect.conf_thresh = saved
    # and one empty image among others: a black frame next to random ones
    frames = mixed_frames(42)
    frames[2] = torch.zeros_like(frames[2])
    check_against_list_path(net, frames, top_k=15)


@pytest.mark.parametrize("config", ["yolact_resnet50_config", "yolact_plus_resnet50_config"])
def test_no_host_sync_and_launches_do_not_grow(config):
    """The launches render_frames adds to infer_frames' (the network's plan may differ with B) are the same for B = 1
    and B = 8, and no call syncs the host."""
    net = net_for(config, "f16x3")
    one, eight, mixed = batch_frames(51, B=1), batch_frames(52, B=8), mixed_frames(53)
    for f in (one, eight, mixed):
        net.render_frames(f, top_k=15, score_threshold=0.15)   # graphs and workspaces exist before counting
    torch.cuda.synchronize()

    def launches(fn):
        n0 = launch_count() + net.launch_count()
        fn()
        return launch_count() + net.launch_count() - n0

    added = [launches(lambda: net.render_frames(f, top_k=15, score_threshold=0.15)) -
             launches(lambda: net.infer_frames(f)) for f in (one, eight)]
    assert added[0] == added[1], added
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        net.render_frames(eight, top_k=15, score_threshold=0.3, fps_box=(60, 14))
        net.render_frames(mixed, top_k=100)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def restated_display(det, frame, top_k, thr, class_color=False, crop_masks=True, mask_alpha=0.45, fps_box=None,
                     draw_masks=True):
    """eval.py:147-224 in torch on the GPU, then `(img_gpu * 255).byte()`: postprocess(rescore_bbox) masks, the stable
    descending order, the top_k rows and the score cut, the reference's blend expression, the fps box
    `img_gpu[0:text_h+8, 0:text_w+8] *= 0.6`.  The dim-0 sum, prod and cumprod of the blend are written out in drawing
    order, the order the kernels evaluate them in.  `/ 255` is true division, as the reference rounds it on the CPU
    (tests/golden) and as the kernels and the palette do: torch's CUDA division by a Python scalar multiplies by the
    reciprocal instead, which rounds differently for 126 of the 256 byte values and 22 of the palette's 47."""
    dets = [{"detection": dict(det) if det is not None else None, "net": None}]
    cfg = ybcfg.cfg
    save, cfg.rescore_bbox = cfg.rescore_bbox, True
    try:
        t = postprocess(dets, int(frame.shape[1]), int(frame.shape[0]), crop_masks=crop_masks, score_threshold=thr,
                        mask_format="u8")
    finally:
        cfg.rescore_bbox = save
    img_gpu = frame.float() / torch.full_like(frame, 255, dtype=torch.float32)   # true division, see the docstring
    n = 0
    if t[1].numel():
        idx = torch.sort(t[1], descending=True, stable=True)[1][:top_k]
        masks, classes, scores = t[3][idx], t[0][idx].cpu().numpy(), t[1][idx].cpu().numpy()
        n = min(top_k, classes.shape[0])
        for j in range(n):
            if scores[j] < thr:
                n = j
                break
    if draw_masks and n > 0:
        masks = masks[:n, :, :, None].float()
        colors = torch.cat([(torch.tensor(get_color(j, classes, class_color, bgr=True), dtype=torch.float32)
                             / 255.).cuda().view(1, 1, 1, 3) for j in range(n)], dim=0)
        masks_color = masks.repeat(1, 1, 1, 3) * colors * mask_alpha
        inv_alph_masks = masks * (-mask_alpha) + 1
        masks_color_summand = masks_color[0]
        if n > 1:
            cumul = [inv_alph_masks[0]]
            for j in range(1, n - 1):
                cumul.append(cumul[-1] * inv_alph_masks[j])
            total = masks_color[1] * cumul[0]
            for j in range(2, n):
                total = total + masks_color[j] * cumul[j - 1]
            masks_color_summand = masks_color_summand + total
        prod = inv_alph_masks[0]
        for j in range(1, n):
            prod = prod * inv_alph_masks[j]
        img_gpu = img_gpu * prod + masks_color_summand
    if fps_box is not None:
        text_w, text_h = fps_box
        img_gpu[0:text_h + 8, 0:text_w + 8] *= 0.6
    return (img_gpu * 255).byte()


@pytest.mark.parametrize("fps_box,draw_masks", [((107, 14), True), ((400, 14), False), ((1, 14), True),
                                                 ((250, 300), True), (None, False), ((0, 14), True)])
def test_fps_box_and_display_masks_match_the_torch_restatement(fps_box, draw_masks):
    ybcfg.set_cfg("yolact_base_config")
    ns = [37, 0, 100, 1]
    dets = [make_dets(n, 138, 138, 600 + i) if n else None for i, n in enumerate(ns)]
    sizes = [(203, 277), (77, 101), (550, 550), (5, 7)]
    for top_k, thr, class_color in ((5, 0, False), (15, 0.15, True), (100, 0.3, False)):
        for dtype in (torch.uint8, torch.float32):
            frames = frames_for(sizes, 7 + top_k, dtype)
            images, _ = render_masks([{"detection": d, "net": None} for d in dets], frames, top_k=top_k,
                                     score_threshold=thr, class_color=class_color, fps_box=fps_box,
                                     draw_masks=draw_masks)
            for i, (d, f) in enumerate(zip(dets, frames)):
                want = restated_display(d, f, top_k, thr, class_color=class_color, fps_box=fps_box,
                                        draw_masks=draw_masks)
                bad = images[i] != want
                assert not bad.any(), (i, top_k, thr, dtype, fps_box, draw_masks, int(bad.sum()),
                                       int((images[i].int() - want.int()).abs().max()))


def test_fps_box_and_display_masks_through_render_frames_match_the_restatement():
    net = net_for("yolact_resnet50_config", "f16x3")
    frames = mixed_frames(61)
    preds = net.forward_frames(frames)
    for fps_box, draw_masks in (((107, 14), True), ((300, 14), False)):
        images, _ = net.render_frames(frames, top_k=5, score_threshold=0.15, fps_box=fps_box, draw_masks=draw_masks)
        for i, f in enumerate(frames):
            want = restated_display(preds[i]["detection"], f, 5, 0.15, fps_box=fps_box, draw_masks=draw_masks)
            assert torch.equal(images[i], want), (i, fps_box, draw_masks)


def golden():
    z = np.load(GOLDEN)
    det = {"box": torch.from_numpy(z["box"]).cuda(), "mask": torch.from_numpy(z["coef"]).cuda(),
           "class": torch.from_numpy(z["cls"]).cuda(), "score": torch.from_numpy(z["score"]).cuda(),
           "proto": torch.from_numpy(z["proto"]).cuda()}
    return z, det


def case_args(z, name):
    top_k, thr_e6, class_color, display_masks, display_text, display_bboxes = (int(v) for v in z[name + "_args"])
    return dict(top_k=top_k, score_threshold=thr_e6 / 1e6, class_color=bool(class_color),
                display_masks=bool(display_masks), display_text=bool(display_text),
                display_bboxes=bool(display_bboxes))


@pytest.mark.parametrize("name", ["video_box", "nomasks_box", "full_box"])
def test_render_matches_the_reference_fps_box_and_display_masks(name):
    """The golden's fps string is spaces, which draw no glyph: its image is prep_display's GPU part alone."""
    ybcfg.set_cfg("yolact_base_config")
    z, det = golden()
    a = case_args(z, name)
    assert not a["display_text"] and not a["display_bboxes"]
    frame = torch.from_numpy(z[name + "_frame"]).cuda()
    for f in (frame, frame.float()):
        images, _ = render_masks([{"detection": det, "net": None}], [f], top_k=a["top_k"],
                                 score_threshold=a["score_threshold"], class_color=a["class_color"],
                                 fps_box=tuple(int(v) for v in z[name + "_fps_wh"]), draw_masks=a["display_masks"])
        diff = np.abs(images[0].cpu().numpy().astype(np.int32) - z[name + "_out"].astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 2e-3, (name, diff.max(), (diff > 0).mean())


@pytest.mark.parametrize("name", ["video", "nomasks", "full"])
def test_install_display_matches_the_reference_full_display(name):
    """install_display's prep_display on a fake eval module: masks, fps box, fps text, boxes and labels."""
    pytest.importorskip("cv2")
    from integration.use_b200 import install_display
    ybcfg.set_cfg("yolact_base_config")
    z, det = golden()
    a = case_args(z, name)

    def original(*args, **kw):
        raise AssertionError("the display modes must not reach the original prep_display")

    args = types.SimpleNamespace(top_k=a["top_k"], score_threshold=a["score_threshold"], crop=True,
                                 display_masks=a["display_masks"], display_fps=True, display_text=a["display_text"],
                                 display_bboxes=a["display_bboxes"], display_scores=True, display_lincomb=False)
    E = types.SimpleNamespace(args=args, prep_display=original,
                              cfg=types.SimpleNamespace(eval_mask_branch=True, rescore_bbox=False,
                                                        dataset=types.SimpleNamespace(
                                                            class_names=tuple(str(c) for c in z["coco_classes"]))))
    install_display(E)
    frame = torch.from_numpy(z[name + "_frame"]).cuda().float()   # evalimage / evalvideo: .cuda().float()
    out = E.prep_display([{"detection": dict(det), "net": None}], frame, None, None, undo_transform=False,
                         class_color=a["class_color"], fps_str=str(z[name + "_fps_str"]))
    assert isinstance(out, np.ndarray) and out.dtype == np.uint8
    diff = np.abs(out.astype(np.int32) - z[name + "_out"].astype(np.int32))
    assert (diff > 1).mean() < 2e-3 and (diff > 0).mean() < 2e-3, (name, (diff > 1).mean(), (diff > 0).mean())


def test_c_abi_ex_rejects_bad_options_and_writes_nothing():
    ybcfg.set_cfg("yolact_base_config")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = _ops_handle(dev, 32)
    d = make_dets(6, 138, 138, 70)
    frame = frames_for([(20, 30)], 71, torch.uint8)[0]
    out = torch.full_like(frame, 7)
    sel_n = torch.full((1,), -5, dtype=torch.int32, device=dev)
    sel_cls = torch.full((5,), -5, dtype=torch.int64, device=dev)
    counts = torch.tensor([4], dtype=torch.int32, device=dev)
    host_counts = np.array([4], np.int32)
    pal = _palette(dev)

    def item(**over):
        it = _lib.YbRenderItem(frame.data_ptr(), out.data_ptr(), d["proto"].data_ptr(), d["mask"].data_ptr(),
                               d["box"].data_ptr(), d["class"].data_ptr(), d["score"].data_ptr(), d["score"].data_ptr(),
                               sel_n.data_ptr(), sel_cls.data_ptr(), None, None, 6, 20, 30)
        for k, v in over.items():
            setattr(it, k, v)
        return it

    def call(it, opts, top_k=5):
        items = (_lib.YbRenderItem * 1)(it)
        return lib.yb_render_list_ex(h, items, 1, 1, 138, 138, 32, 1, top_k, 0.0, 0, 0.45, _lib.ptr(pal),
                                     len(ybcfg.COLORS), opts, _lib.current_stream(dev))

    def opts(**over):
        o = _lib.YbRenderOpts(counts.data_ptr(), 10, 4, 1)
        for k, v in over.items():
            setattr(o, k, v)
        return o

    refusals = [(item(), opts(fps_w=-1)), (item(), opts(fps_h=-3)), (item(), opts(d_counts=host_counts.ctypes.data)),
                (item(frame=None), opts()), (item(n=-1), opts()), (item(cls=None), opts())]
    for it, o in refusals:
        assert call(it, o) == YB_ERR_INVALID, (o.fps_w, o.fps_h)
        assert lib.yb_last_error()
    assert call(item(), opts(), top_k=0) == YB_ERR_INVALID
    torch.cuda.synchronize()
    assert (out == 7).all() and int(sel_n) == -5 and (sel_cls == -5).all()   # nothing was written
    assert call(item(), None) == 0, lib.yb_last_error()                       # NULL options: yb_render_list
    assert call(item(), opts()) == 0, lib.yb_last_error()
    torch.cuda.synchronize()
    assert int(sel_n) == 4   # at most the device count of the 6 rows
