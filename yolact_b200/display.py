"""The GPU part of prep_display (eval.py:135-262) for a list of frames, straight from the detections.

    images, drawn = render_masks(det_output, frames, top_k=5, score_threshold=0, class_color=False,
                                 mask_alpha=0.45, crop_masks=True)

For frame i, images[i] equals prep_display(det_output[i:i+1], frames[i], None, None, undo_transform=False) with
display_text and display_bboxes off: postprocess with cfg.rescore_bbox = True (YOLACT++ ranks by score * maskiou), the
score filter, a stable descending sort (ties to the lower row), the first top_k rows, the cut at the first score below
score_threshold, the palette, the mask blend and `(img_gpu * 255).byte()`.  `drawn` holds the drawn rows -- device
tensors num [B] int32, classes [B,top_k] int64, scores [B,top_k] float32 and boxes [B,top_k,4] int64 pixel boxes, zero
past num -- so that the caller's OpenCV text and rectangles (eval.py:233-259) need one device-to-host copy.

The masks are never written: one selection launch and one render launch cover the whole list, and each output pixel
evaluates only the drawn detections whose crop window reaches it.  YOLACT++'s maskiou_net runs once over the rows of all
images.  There is no host sync at any score_threshold, and there is no CPU path.
"""
import torch

from . import _lib
from . import config as _config
from .output_utils import _maskiou_rescore, _ops_handle

_palettes = {}


def _palette(dev):
    """COLORS as fp32 0..1 BGR [P,3] on dev: the values get_color(...) / 255.0 gives prep_display (eval.py:169-183)."""
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _palettes:
        host = torch.tensor([[c[2] / 255.0, c[1] / 255.0, c[0] / 255.0] for c in _config.COLORS], dtype=torch.float32)
        _palettes[key] = host.pin_memory().to(dev, non_blocking=True)
    return _palettes[key]


def render_masks(det_output, frames, top_k=5, score_threshold=0, class_color=False, mask_alpha=0.45, crop_masks=True):
    """frames: a list of CUDA [h_i,w_i,3] BGR tensors or one [B,h,w,3] tensor, uint8 or float32 0..255, one per entry of
    det_output (Yolact's output list).  Returns (images, drawn): images a list of CUDA uint8 [h_i,w_i,3]; drawn a dict
    of device tensors num, classes, scores, boxes (see the module docstring)."""
    if isinstance(frames, torch.Tensor):
        if frames.dim() != 4:
            raise ValueError("render_masks: a frame tensor must be [B,h,w,3], got %s" % (tuple(frames.shape),))
        frames = list(frames.unbind(0))
    frames = list(frames)
    if len(frames) != len(det_output):
        raise ValueError("render_masks: %d frames for %d detections" % (len(frames), len(det_output)))
    top_k = int(top_k)
    if top_k < 1:
        raise ValueError("render_masks: top_k must be >= 1")
    for f in frames:
        if not f.is_cuda:
            raise _lib.YbError("yolact_b200.render_masks runs on CUDA (H100) only; there is no CPU path.")
        if f.dim() != 3 or f.shape[2] != 3 or f.shape[0] == 0 or f.shape[1] == 0:
            raise ValueError("render_masks: frames must be [h,w,3], got %s" % (tuple(f.shape),))
    dtypes = {f.dtype for f in frames}
    if not dtypes <= {torch.uint8, torch.float32} or len(dtypes) > 1:
        raise ValueError("render_masks: frames must all be uint8 or all float32, got %s" % sorted(map(str, dtypes)))
    B = len(frames)
    dev = frames[0].device if B else torch.device("cuda", torch.cuda.current_device())
    drawn = {"num": torch.zeros(B, dtype=torch.int32, device=dev),
             "classes": torch.zeros(B, top_k, dtype=torch.int64, device=dev),
             "scores": torch.zeros(B, top_k, dtype=torch.float32, device=dev),
             "boxes": torch.zeros(B, top_k, 4, dtype=torch.int64, device=dev)}
    if B == 0:
        return [], drawn
    frames = [f.contiguous() for f in frames]
    images = [torch.empty(int(f.shape[0]), int(f.shape[1]), 3, dtype=torch.uint8, device=dev) for f in frames]

    cfg = _config.cfg
    live = [i for i, d in enumerate(det_output) if d['detection'] is not None]
    dets = {i: det_output[i]['detection'] for i in live}
    for d in dets.values():
        if not d['box'].is_cuda:
            raise _lib.YbError("yolact_b200.render_masks runs on CUDA (H100) only; there is no CPU path.")
    with_proto = ['proto' in d for d in dets.values()]
    if any(with_proto) and not all(with_proto):
        raise ValueError("render_masks: some detections carry 'proto' and some do not")
    eval_mask_branch = bool(live) and getattr(cfg, "eval_mask_branch", True) and with_proto[0]
    keep_alive = []   # the contiguous inputs, held until the calls have enqueued their reads of them
    ph = pw = 1
    k = 4
    rank = {i: dets[i]['score'] for i in live}
    if eval_mask_branch:
        shapes = {tuple(int(s) for s in d['proto'].shape) for d in dets.values()}
        if len(shapes) != 1:
            raise ValueError("render_masks: the images' prototypes differ in (ph, pw, k): %s" % sorted(shapes))
        ph, pw, k = shapes.pop()
        net = det_output[live[0]]['net']
        ncfg = getattr(net, "cfg", cfg)
        if bool(getattr(ncfg, "use_maskiou", False)):
            # YOLACT++ (output_utils.py:77-88 with rescore_bbox, eval.py:148-149): maskiou_net on the prototype-resolution
            # masks of every row of every image at once; the rows are independent, so the score filter can follow
            if any(det_output[i]['net'] is not net for i in live):
                raise ValueError("render_masks: maskiou rescoring needs every image to come from the same net")
            ns = [int(dets[i]['box'].shape[0]) for i in live]
            pm = torch.empty(sum(ns), ph, pw, dtype=torch.float32, device=dev)
            items = (_lib.YbPostItem * len(live))()
            off = 0
            for j, (i, n) in enumerate(zip(live, ns)):
                d = dets[i]
                proto, coef, box = d['proto'].contiguous().float(), d['mask'].contiguous().float(), d['box'].contiguous().float()
                keep_alive += [proto, coef, box]
                items[j] = _lib.YbPostItem(proto.data_ptr(), coef.data_ptr(), box.data_ptr(), None, None,
                                           pm[off:off + n].data_ptr() if n else None, n, int(frames[i].shape[0]),
                                           int(frames[i].shape[1]))
                off += n
            lib = _lib.load()
            _lib.check(lib.yb_postprocess_list(_ops_handle(dev, k), items, len(live), ph, pw, k, 1 if crop_masks else 0,
                                               _lib.YB_MASK_F32, _lib.current_stream(dev)), "yb_postprocess_list(proto)")
            if off > 0:
                cat = (lambda ts: torch.cat(ts)) if len(live) > 1 else (lambda ts: ts[0])
                rescored = _maskiou_rescore(net, ncfg, pm, cat([dets[i]['class'] for i in live]),
                                            cat([dets[i]['score'] for i in live]))
                if rescored is not None:
                    off = 0
                    for i, n in zip(live, ns):
                        rank[i] = rescored[0][off:off + n]
                        off += n

    items = (_lib.YbRenderItem * B)()
    num, classes, scores, boxes = drawn["num"], drawn["classes"], drawn["scores"], drawn["boxes"]
    for i, f in enumerate(frames):
        h, w = int(f.shape[0]), int(f.shape[1])
        it = _lib.YbRenderItem()
        it.frame, it.out = f.data_ptr(), images[i].data_ptr()
        it.sel_n, it.sel_cls = num[i:].data_ptr(), classes[i].data_ptr()
        it.sel_score, it.sel_box = scores[i].data_ptr(), boxes[i].data_ptr()
        it.h, it.w = h, w
        d = dets.get(i)
        n = int(d['box'].shape[0]) if d is not None else 0
        if n > 0:
            box = d['box'].contiguous().float()
            cls = d['class'].contiguous().long()
            det_score = d['score'].contiguous().float()
            score = rank[i].contiguous().float()
            keep_alive += [box, cls, det_score, score]
            it.box, it.cls, it.det_score, it.score = box.data_ptr(), cls.data_ptr(), det_score.data_ptr(), score.data_ptr()
            if eval_mask_branch:
                proto, coef = d['proto'].contiguous().float(), d['mask'].contiguous().float()
                keep_alive += [proto, coef]
                it.proto, it.coef = proto.data_ptr(), coef.data_ptr()
        it.n = n
        items[i] = it
    lib = _lib.load()
    _lib.check(lib.yb_render_list(_ops_handle(dev, k), items, B, 1 if frames[0].dtype == torch.uint8 else 0, ph, pw, k,
                                  1 if crop_masks else 0, top_k, float(score_threshold), 1 if class_color else 0,
                                  float(mask_alpha), _lib.ptr(_palette(dev)), len(_config.COLORS),
                                  _lib.current_stream(dev)), "yb_render_list")
    return images, drawn
