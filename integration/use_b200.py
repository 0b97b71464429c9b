"""Route the reference's eval.py through the H100 path without editing a line of it (INTEGRATION.md section 1).

    import integration.use_b200 as ub
    ub.install("/path/to/yolact")          # BEFORE `import eval`
    import eval as E                        # the reference's eval.py, unchanged
    E.parse_args([...]); ... E.evaluate(net, dataset)

or, from the shell:   python -m integration.use_b200 /path/to/yolact --trained_model=... --benchmark

For the mAP mode, `install_metrics(E)` after `import eval as E` also moves prep_metrics' matching loop and calc_map to
the GPU (yolact_b200.metrics); `install_coco_json(E)` does the same for --output_coco_json's records, and
`install_display(E)` routes --image, --images and --video frames' prep_display through yolact_b200.display.  The shell
route runs eval.py as a fresh `__main__` module that cannot be patched, so it keeps the reference's own loop.

`install` puts the reference on sys.path, imports its modules and rebinds the names eval.py pulls from them
(`from yolact import Yolact`, `from layers.output_utils import postprocess`, `from utils.augmentations import
FastBaseTransform`, `from layers.box_utils import jaccard, mask_iou`) to this package's mirrors.  The reference `cfg`
stays the object eval.py mutates; it is snapshotted into yolact_b200.cfg each time a Yolact is constructed
(eval.py calls set_cfg before `Yolact()`, eval.py:1085-1097).
"""
import sys

# cfg keys the reference's callers flip on the GLOBAL cfg between calls (prep_display sets rescore_bbox = True around
# postprocess, eval.py:147-151; --detect clears eval_mask_branch, eval.py:1074): the package snapshot would go stale,
# so every routed call re-reads them from the live reference cfg.
LIVE_CFG_KEYS = ("rescore_bbox", "rescore_mask", "eval_mask_branch", "mask_proto_debug")


def _refresh_cfg(ref_cfg):
    """Copies LIVE_CFG_KEYS that ref_cfg (a reference cfg object) has into yolact_b200.cfg."""
    import yolact_b200
    for key in LIVE_CFG_KEYS:
        if hasattr(ref_cfg, key):
            setattr(yolact_b200.cfg, key, getattr(ref_cfg, key))


def install(reference_root, mask_iou_on_gpu=True):
    if reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    import yolact_b200
    from yolact_b200 import eval_utils
    from yolact_b200.config import from_reference_cfg
    from yolact_b200.augmentations import FastBaseTransform as B200FastBaseTransform

    import data as ref_data                      # noqa: the reference's packages
    import yolact as ref_yolact
    import layers.output_utils as ref_output_utils
    import layers.box_utils as ref_box_utils
    import utils.augmentations as ref_aug

    class Yolact(yolact_b200.Yolact):
        """`Yolact()` with the reference's no-argument constructor: reads the reference's global cfg."""

        def __init__(self):
            yolact_b200.cfg.replace(from_reference_cfg(ref_data.cfg))
            super().__init__()

    class FastBaseTransform(B200FastBaseTransform):
        def __init__(self):
            super().__init__(from_reference_cfg(ref_data.cfg))

    def postprocess(*args, **kwargs):
        _refresh_cfg(ref_data.cfg)
        return yolact_b200.postprocess(*args, **kwargs)
    postprocess.__doc__ = yolact_b200.postprocess.__doc__

    ref_yolact.ReferenceYolact = ref_yolact.Yolact          # the PyTorch graph stays reachable
    ref_yolact.Yolact = Yolact
    ref_output_utils.postprocess = postprocess
    ref_aug.FastBaseTransform = FastBaseTransform
    if mask_iou_on_gpu:
        ref_box_utils.mask_iou = eval_utils.mask_iou
        ref_box_utils.jaccard = eval_utils.jaccard
    return {"Yolact": Yolact, "postprocess": postprocess, "FastBaseTransform": FastBaseTransform}


APDATA_KEY = "_yb_apdata"   # where the GPU accumulator lives inside eval.py's ap_data dict


def install_metrics(E):
    """Rebind E.prep_metrics and E.calc_map (E: the reference's `eval` module, imported after install()) to
    yolact_b200.metrics.  evaluate() keeps building its ap_data dict and passing it around; the patched prep_metrics
    keeps one APData in it under APDATA_KEY ('box' / 'mask' stay as evaluate() made them), so the pickle evaluate()
    writes to --ap_data_file holds the accumulator and reloads for --resume.  --output_coco_json goes to the original
    prep_metrics; the patched calc_map falls back to the original for an ap_data without the key."""
    from yolact_b200 import metrics

    orig_prep, orig_calc = E.prep_metrics, E.calc_map

    def prep_metrics(ap_data, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections=None):
        if E.args.output_coco_json:
            return orig_prep(ap_data, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections)
        apd = ap_data.get(APDATA_KEY)
        if apd is None:
            apd = ap_data[APDATA_KEY] = metrics.APData(len(E.cfg.dataset.class_names), E.iou_thresholds)
        metrics.prep_metrics(apd, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections,
                             crop_masks=E.args.crop, score_threshold=E.args.score_threshold, postprocess=E.postprocess)

    def calc_map(ap_data):
        if not isinstance(ap_data, dict) or APDATA_KEY not in ap_data:
            return orig_calc(ap_data)
        return metrics.calc_map(ap_data[APDATA_KEY])

    prep_metrics.__doc__, calc_map.__doc__ = metrics.prep_metrics.__doc__, metrics.calc_map.__doc__
    E.prep_metrics, E.calc_map = prep_metrics, calc_map
    return {"prep_metrics": prep_metrics, "calc_map": calc_map}


def install_coco_json(E):
    """Wrap whatever E.prep_metrics is bound to now (the reference's, or install_metrics'; either install order works)
    so that with --output_coco_json its records come from yolact_b200.metrics.Detections' GPU route: one
    yb_coco_rle_list launch per image instead of full-size fp32 masks and pycocotools on the host.  The records are
    appended to the reference's own `detections` object (bbox_data / mask_data, categories from E.get_coco_cat), so
    evaluate()'s detections.dump() and dump_web() run unchanged.  Without the flag the call goes to the previous
    binding."""
    from yolact_b200 import metrics

    prev = E.prep_metrics

    def prep_metrics(ap_data, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections=None):
        if not E.args.output_coco_json:
            return prev(ap_data, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections)
        _refresh_cfg(getattr(E, "cfg", None))
        sink = metrics.Detections(E.get_coco_cat)
        sink.bbox_data, sink.mask_data = detections.bbox_data, detections.mask_data
        sink.add(dets[:1], [(h, w)], [image_id], crop_masks=E.args.crop, score_threshold=E.args.score_threshold)

    prep_metrics.__doc__ = install_coco_json.__doc__
    E.prep_metrics = prep_metrics
    return {"prep_metrics": prep_metrics}


def install_display(E):
    """Rebind E.prep_display (eval.py:135-262) so that --image, --images and --video frames, the calls with
    undo_transform=False, take yolact_b200.display.render_masks: the rows are selected and the masks blended straight
    from the detections in two launches, with the --display_fps box and --display_masks, instead of postprocess writing
    fp32 masks for every row at frame size.  The image and the drawn rows come to the host in one copy, and the fps
    text, rectangles and labels are drawn on it with OpenCV from the drawn rows, as eval.py:226-259 draws them.
    Detections on another GPU than the frame (a CustomDataParallel replica's, evalvideo) are copied to the frame's
    device first, and the image is that of the same-device render.
    undo_transform=True (evaluate --display) and --display_lincomb go to the original prep_display."""
    import torch
    from yolact_b200 import display
    from yolact_b200.eval_utils import get_color

    orig = E.prep_display

    def prep_display(dets_out, img, h, w, undo_transform=True, class_color=False, mask_alpha=0.45, fps_str=''):
        args = E.args
        if undo_transform or args.display_lincomb:
            return orig(dets_out, img, h, w, undo_transform=undo_transform, class_color=class_color,
                        mask_alpha=mask_alpha, fps_str=fps_str)
        import cv2
        _refresh_cfg(getattr(E, "cfg", None))
        font_face, font_scale, font_thickness = cv2.FONT_HERSHEY_DUPLEX, 0.6, 1
        text_w = text_h = 0
        if args.display_fps:
            text_w, text_h = cv2.getTextSize(fps_str, font_face, font_scale, font_thickness)[0]
        images, drawn = display.render_masks(dets_out[:1], [img], top_k=args.top_k,
                                             score_threshold=args.score_threshold, class_color=class_color,
                                             mask_alpha=mask_alpha, crop_masks=args.crop,
                                             fps_box=(text_w, text_h) if args.display_fps else None,
                                             draw_masks=args.display_masks)
        # one copy to the host: the image and the drawn rows, enqueued together, then one wait
        dev = images[0].device
        host = [t.to("cpu", non_blocking=True) for t in (images[0], drawn["num"][0], drawn["classes"][0],
                                                            drawn["scores"][0], drawn["boxes"][0])]
        if dev.type == "cuda":
            torch.cuda.current_stream(dev).synchronize()
        img_numpy, num, classes, scores, boxes = (t.numpy() for t in host)

        if args.display_fps:
            cv2.putText(img_numpy, fps_str, (4, text_h + 2), font_face, font_scale, [255, 255, 255], font_thickness,
                        cv2.LINE_AA)
        num = int(num)
        if num == 0 or not (args.display_text or args.display_bboxes):
            return img_numpy
        for j in reversed(range(num)):
            x1, y1, x2, y2 = (int(v) for v in boxes[j])
            color = get_color(j, classes, class_color, bgr=True)
            if args.display_bboxes:
                cv2.rectangle(img_numpy, (x1, y1), (x2, y2), color, 1)
            if args.display_text:
                _class = E.cfg.dataset.class_names[classes[j]]
                text_str = '%s: %.2f' % (_class, scores[j]) if args.display_scores else _class
                tw, th = cv2.getTextSize(text_str, font_face, font_scale, font_thickness)[0]
                cv2.rectangle(img_numpy, (x1, y1), (x1 + tw, y1 - th - 4), color, -1)
                cv2.putText(img_numpy, text_str, (x1, y1 - 3), font_face, font_scale, [255, 255, 255], font_thickness,
                            cv2.LINE_AA)
        return img_numpy

    prep_display.__doc__ = install_display.__doc__
    E.prep_display = prep_display
    return {"prep_display": prep_display}


if __name__ == "__main__":
    import runpy
    root = sys.argv[1]
    install(root)
    sys.argv = [root + "/eval.py"] + sys.argv[2:]
    runpy.run_path(root + "/eval.py", run_name="__main__")   # the reference's eval.py, as its own __main__
