"""Generates tests/golden/display_unit.npz: eval.py's prep_display for the --image / --images / --video display modes,
run by the REAL reference on the CPU.

    python scripts/gen_display_golden.py      # needs the reference checkout at REF

Runs the reference's own prep_display (eval.py:135-262) with undo_transform=False on a BGR frame 0..255, as evalimage
and evalvideo call it.  Shims, never edits to the reference: stub pycocotools / matplotlib modules, a Tensor subclass
whose `.device.index` is 0 and Tensor.to(int) as the identity, because the reference only takes its GPU colour path when
the image reports a CUDA device (eval.py:171-183,193).

Cases (display_unit.npz keys `<case>_*`):
  video      evalvideo's call: class_color=True, --display_fps with an fps string wider than the narrow frame (the box
             is clipped), text and boxes on;
  video_box  the same with an fps string of spaces and text and boxes off: the fps box and the mask blend alone (the
             spaces draw no pixel), so the GPU part is pinned without OpenCV's glyphs;
  nomasks    --display_masks=False with the fps box, text and boxes on;
  nomasks_box  --display_masks=False with the box of spaces, text and boxes off;
  full       the default full display (top_k 5, score_threshold 0.15, text and boxes) with the fps box;
  full_box   its masks and box of spaces, text and boxes off.
Per case: `frame` (uint8), `args` (top_k, score_threshold * 1e6, class_color, display_masks, display_text,
display_bboxes), `fps_str`, `fps_wh` (cv2.getTextSize of it), `out` (prep_display's uint8 image).  The detections
(`proto`, `coef`, `box`, `score`, `cls`) are shared, with `coco_classes`.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "display_unit.npz")


def install_shims():
    for m in ["pycocotools", "pycocotools.mask", "pycocotools.coco", "pycocotools.cocoeval", "matplotlib",
              "matplotlib.pyplot"]:
        sys.modules.setdefault(m, types.ModuleType(m))
    sys.modules["pycocotools.coco"].COCO = object
    torch.cuda.current_device = lambda: 0
    if REF not in sys.path:
        sys.path.insert(0, REF)


class _OnGpu0(torch.Tensor):
    @property
    def device(self):
        return types.SimpleNamespace(index=0)


def main():
    install_shims()
    import cv2
    import eval as E
    from data.config import cfg, set_cfg
    set_cfg("yolact_base_config")
    cfg.mask_proto_debug = False

    r = np.random.RandomState(29)
    # prototypes and coefficients on coarse grids (eighths, sixteenths): the values stay exact in fp32 and the file small
    n, ph, pw, K = 14, 48, 48, 32
    proto = np.maximum(r.standard_normal((ph, pw, K)), 0).astype(np.float32)
    proto = (proto + np.roll(proto, 1, 0) + np.roll(proto, 1, 1) + np.roll(proto, (2, 3), (0, 1))) / 4
    proto = (np.round(proto * 8) / 8).astype(np.float32)
    coef = (np.round(np.tanh(r.standard_normal((n, K))) * 16) / 16).astype(np.float32)
    c = r.uniform(0.2, 0.8, (n, 2))
    wh = r.uniform(0.1, 0.6, (n, 2))
    box = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(np.float32)
    box[0] = [0.0, 0.0, 0.45, 0.4]       # the top scorer covers the fps box's corner
    score = np.sort(r.uniform(0.05, 0.99, n).astype(np.float32))[::-1].copy()
    cls = r.randint(0, 80, n).astype(np.int64)

    def frame(h, w):   # random colours in 8 x 8 blocks: the values cover 0..255, and the file stays small
        blocks = r.randint(0, 256, ((h + 7) // 8, (w + 7) // 8, 3)).astype(np.uint8)
        return np.ascontiguousarray(blocks.repeat(8, 0).repeat(8, 1)[:h, :w])

    narrow, wide = frame(150, 96), frame(203, 277)
    spaces = " " * 12
    fps_long = "FPS: 29.97 (1920x1080)"
    # name: (frame, argv, prep_display kwargs, fps_str)
    cases = {
        "video": (narrow, [], dict(class_color=True), fps_long),
        "video_box": (narrow, ["--display_text=False", "--display_bboxes=False"], dict(class_color=True), spaces * 3),
        "nomasks": (wide, ["--display_masks=False", "--score_threshold=0.15"], {}, "FPS: 7.50"),
        "nomasks_box": (wide, ["--display_masks=False", "--display_text=False", "--display_bboxes=False"], {}, spaces),
        "full": (wide, ["--top_k=5", "--score_threshold=0.15"], {}, "FPS: 12.34"),
        "full_box": (wide, ["--top_k=5", "--score_threshold=0.15", "--display_text=False", "--display_bboxes=False"],
                     {}, spaces),
    }
    out = {"proto": proto, "coef": coef, "box": box, "score": score, "cls": cls,
           "coco_classes": np.array(list(cfg.dataset.class_names))}
    orig_to = torch.Tensor.to

    def to_shim(self, *a, **k):
        if a and isinstance(a[0], int):
            return self
        return orig_to(self, *a, **k)

    torch.Tensor.to = to_shim
    try:
        for name, (frame, argv, kw, fps_str) in cases.items():
            E.parse_args(argv + ["--display_fps"])
            E.color_cache.clear()
            a = E.args
            if fps_str.strip() == "":
                # the box of spaces draws no glyph: the output is prep_display's GPU part alone
                probe = np.zeros((40, 400, 3), np.uint8)
                cv2.putText(probe, fps_str, (4, 16), cv2.FONT_HERSHEY_DUPLEX, 0.6, [255, 255, 255], 1, cv2.LINE_AA)
                assert not probe.any()
            det = {"box": torch.from_numpy(box.copy()), "mask": torch.from_numpy(coef.copy()),
                   "class": torch.from_numpy(cls.copy()), "score": torch.from_numpy(score.copy()),
                   "proto": torch.from_numpy(proto.copy())}
            img = torch.from_numpy(frame.astype(np.float32)).as_subclass(_OnGpu0)
            with torch.no_grad():
                res = E.prep_display([{"detection": det, "net": None}], img, None, None, undo_transform=False,
                                     fps_str=fps_str, **kw)
            fps_wh = cv2.getTextSize(fps_str, cv2.FONT_HERSHEY_DUPLEX, 0.6, 1)[0]
            out[name + "_frame"] = frame
            out[name + "_args"] = np.array([a.top_k, round(a.score_threshold * 1e6), int(kw.get("class_color", False)),
                                            int(a.display_masks), int(a.display_text), int(a.display_bboxes)], np.int64)
            out[name + "_fps_str"] = np.array(fps_str)
            out[name + "_fps_wh"] = np.array(fps_wh, np.int64)
            out[name + "_out"] = np.asarray(res)
            print(name, res.shape, "fps box", fps_wh, "mean %.2f" % np.asarray(res).mean())
    finally:
        torch.Tensor.to = orig_to
    np.savez_compressed(OUT, **out)
    print("wrote %s (%.2f MB)" % (OUT, os.path.getsize(OUT) / 1e6))


if __name__ == "__main__":
    main()
