"""integration.use_b200.install_display's routing, on the CPU: a fake eval module and a fake renderer stand in for eval.py
and yolact_b200.display.render_masks.  Which calls reach the renderer, with which arguments (eval.py's args, and the fps
box from cv2.getTextSize of the fps string), which go to the original prep_display, and what is drawn on the host from
the drawn rows."""
import types

import numpy as np
import pytest
import torch

import yolact_b200
from integration.use_b200 import install_display
from yolact_b200 import display
from yolact_b200.eval_utils import get_color

cv2 = pytest.importorskip("cv2")

NAMES = tuple("class%d" % i for i in range(80))


def fake_eval(**over):
    args = dict(top_k=7, score_threshold=0.25, crop=False, display_masks=True, display_fps=False, display_text=False,
                display_bboxes=False, display_scores=True, display_lincomb=False)
    args.update(over)
    calls = []

    def orig(*a, **k):
        calls.append((a, k))
        return "original"

    E = types.SimpleNamespace(args=types.SimpleNamespace(**args), prep_display=orig,
                              cfg=types.SimpleNamespace(eval_mask_branch=True, rescore_bbox=False,
                                                        dataset=types.SimpleNamespace(class_names=NAMES)))
    install_display(E)
    return E, calls


class FakeRenderer:
    """Returns a fixed image and two drawn rows; records each call."""

    def __init__(self, h=60, w=80):
        self.calls = []
        self.image = torch.from_numpy(np.random.RandomState(3).randint(0, 256, (h, w, 3)).astype(np.uint8))
        self.drawn = {"num": torch.tensor([2], dtype=torch.int32),
                      "classes": torch.tensor([[5, 17, 0]]),
                      "scores": torch.tensor([[0.875, 0.3125, 0.0]]),
                      "boxes": torch.tensor([[[10, 30, 40, 55], [2, 20, 70, 50], [0, 0, 0, 0]]])}

    def __call__(self, det_output, frames, **kw):
        self.calls.append((det_output, frames, kw))
        return [self.image.clone()], self.drawn


@pytest.fixture
def renderer(monkeypatch):
    r = FakeRenderer()
    monkeypatch.setattr(display, "render_masks", r)
    return r


def test_undo_transform_and_lincomb_go_to_the_original(renderer):
    E, calls = fake_eval()
    assert E.prep_display(["dets"], "img", 10, 20) == "original"          # undo_transform defaults to True
    assert calls[-1] == ((["dets"], "img", 10, 20), dict(undo_transform=True, class_color=False, mask_alpha=0.45,
                                                         fps_str=''))
    E, calls = fake_eval(display_lincomb=True)
    assert E.prep_display(["dets"], "img", None, None, undo_transform=False, fps_str="x") == "original"
    assert calls[-1][1]["undo_transform"] is False and calls[-1][1]["fps_str"] == "x"
    assert not renderer.calls


@pytest.mark.parametrize("class_color", [False, True])
def test_arguments_reach_the_renderer(renderer, class_color):
    E, calls = fake_eval(display_masks=False)
    frame = torch.zeros(60, 80, 3)
    dets = [{"detection": None, "net": None}, {"detection": "second", "net": None}]
    out = E.prep_display(dets, frame, None, None, undo_transform=False, class_color=class_color, mask_alpha=0.3)
    assert not calls and len(renderer.calls) == 1
    det_output, frames, kw = renderer.calls[0]
    assert det_output == dets[:1] and len(frames) == 1 and frames[0] is frame
    assert kw == dict(top_k=7, score_threshold=0.25, class_color=class_color, mask_alpha=0.3, crop_masks=False,
                      fps_box=None, draw_masks=False)
    assert np.array_equal(out, renderer.image.numpy())   # nothing drawn on the host without text, boxes or fps


def test_the_reference_cfg_is_read_on_every_call(renderer):
    E, _ = fake_eval()
    saved = yolact_b200.cfg.eval_mask_branch
    try:
        E.cfg.eval_mask_branch = False
        E.prep_display([{"detection": None, "net": None}], torch.zeros(4, 4, 3), None, None, undo_transform=False)
        assert yolact_b200.cfg.eval_mask_branch is False
    finally:
        yolact_b200.cfg.eval_mask_branch = saved


@pytest.mark.parametrize("fps_str", ["", "FPS: 29.97", "FPS: 1234.56 at 1920x1080"])
def test_fps_box_and_text(renderer, fps_str):
    E, _ = fake_eval(display_fps=True)
    out = E.prep_display([{"detection": None, "net": None}], torch.zeros(60, 80, 3), None, None,
                         undo_transform=False, fps_str=fps_str)
    text_w, text_h = cv2.getTextSize(fps_str, cv2.FONT_HERSHEY_DUPLEX, 0.6, 1)[0]
    assert renderer.calls[-1][2]["fps_box"] == (text_w, text_h)
    assert text_w >= 1 and text_h == 14   # never (0, 0): an empty string still draws eval.py's box
    want = renderer.image.numpy().copy()
    cv2.putText(want, fps_str, (4, text_h + 2), cv2.FONT_HERSHEY_DUPLEX, 0.6, [255, 255, 255], 1, cv2.LINE_AA)
    assert np.array_equal(out, want)


@pytest.mark.parametrize("text,bboxes,scores", [(True, True, True), (True, False, False), (False, True, True)])
def test_text_and_boxes_are_drawn_from_the_drawn_rows(renderer, text, bboxes, scores):
    """eval.py:236-259 on the renderer's image, from the drawn rows, in reverse drawing order."""
    E, _ = fake_eval(display_text=text, display_bboxes=bboxes, display_scores=scores)
    out = E.prep_display([{"detection": "d", "net": None}], torch.zeros(60, 80, 3), None, None, undo_transform=False,
                         class_color=True)
    want = renderer.image.numpy().copy()
    classes = renderer.drawn["classes"][0].numpy()
    for j in (1, 0):
        x1, y1, x2, y2 = (int(v) for v in renderer.drawn["boxes"][0, j])
        color = get_color(j, classes, True, bgr=True)
        if bboxes:
            cv2.rectangle(want, (x1, y1), (x2, y2), color, 1)
        if text:
            s = '%s: %.2f' % (NAMES[classes[j]], renderer.drawn["scores"][0, j].item()) if scores else NAMES[classes[j]]
            tw, th = cv2.getTextSize(s, cv2.FONT_HERSHEY_DUPLEX, 0.6, 1)[0]
            cv2.rectangle(want, (x1, y1), (x1 + tw, y1 - th - 4), color, -1)
            cv2.putText(want, s, (x1, y1 - 3), cv2.FONT_HERSHEY_DUPLEX, 0.6, [255, 255, 255], 1, cv2.LINE_AA)
    assert np.array_equal(out, want)
    assert not np.array_equal(out, renderer.image.numpy())
