"""The GPU part of prep_display (eval.py:135-262) for a list of frames, straight from the detections.

    images, drawn = render_masks(det_output, frames, top_k=5, score_threshold=0, class_color=False,
                                 mask_alpha=0.45, crop_masks=True, fps_box=None, draw_masks=True)
    images, drawn = net.render_frames(frames, ...)     # the same from uint8 frames, with no host sync (render_frames)

For frame i, images[i] equals prep_display(det_output[i:i+1], frames[i], None, None, undo_transform=False) with
display_text and display_bboxes off: postprocess with cfg.rescore_bbox = True (YOLACT++ ranks by score * maskiou), the
score filter, a stable descending sort (ties to the lower row), the first top_k rows, the cut at the first score below
score_threshold, the palette, the mask blend and `(img_gpu * 255).byte()`.  `drawn` holds the drawn rows -- device
tensors num [B] int32, classes [B,top_k] int64, scores [B,top_k] float32 and boxes [B,top_k,4] int64 pixel boxes, zero
past num -- so that the caller's OpenCV text and rectangles (eval.py:233-259) need one device-to-host copy.

fps_box = (text_w, text_h), cv2.getTextSize of the fps string, is --display_fps' box (eval.py:211-219): the pixels of
rows [0, text_h + 8) and columns [0, text_w + 8) are scaled by 0.6 before `* 255`.  draw_masks=False is
--display_masks=False: the rows are selected and `drawn` written, no mask is blended.

The masks are never written: one selection launch and one render launch cover the whole list, and each output pixel
evaluates only the drawn detections whose crop window reaches it.  YOLACT++'s maskiou_net runs once over the rows of all
images.  There is no host sync at any score_threshold, and there is no CPU path.

render_frames runs the network and the render back to back from Yolact.infer_frames' padded outputs: the items point
into the padded tensors and the selection reads each image's row count on the device, so nothing waits for the host
and a caller can have several batches in flight.
"""
import ctypes

import torch

from . import _lib
from . import config as _config
from .output_utils import _gather, _ops_handle, _post_list, _rescore_list

_palettes = {}


def _palette(dev):
    """COLORS as fp32 0..1 BGR [P,3] on dev: the values get_color(...) / 255.0 gives prep_display (eval.py:169-183)."""
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _palettes:
        host = torch.tensor([[c[2] / 255.0, c[1] / 255.0, c[0] / 255.0] for c in _config.COLORS], dtype=torch.float32)
        _palettes[key] = host.pin_memory().to(dev, non_blocking=True)
    return _palettes[key]


def _frame_list(frames, where):
    """frames ([B,h,w,3] or a sequence of [h,w,3]) as a list."""
    if isinstance(frames, torch.Tensor):
        if frames.dim() != 4:
            raise ValueError("%s: a frame tensor must be [B,h,w,3], got %s" % (where, tuple(frames.shape)))
        frames = list(frames.unbind(0))
    return list(frames)


def _checked_frames(frames, where):
    """The list as contiguous CUDA [h,w,3] tensors, all uint8 or all float32, and their device."""
    for f in frames:
        if not f.is_cuda:
            raise _lib.YbError("yolact_b200.%s runs on CUDA (H100) only; there is no CPU path." % where)
        if f.dim() != 3 or f.shape[2] != 3 or f.shape[0] == 0 or f.shape[1] == 0:
            raise ValueError("%s: frames must be [h,w,3], got %s" % (where, tuple(f.shape)))
    dtypes = {f.dtype for f in frames}
    if not dtypes <= {torch.uint8, torch.float32} or len(dtypes) > 1:
        raise ValueError("%s: frames must all be uint8 or all float32, got %s" % (where, sorted(map(str, dtypes))))
    dev = frames[0].device if frames else torch.device("cuda", torch.cuda.current_device())
    return [f.contiguous() for f in frames], dev


def _opts(fps_box, draw_masks):
    """yb_render_opts for fps_box = None or (text_w, text_h) and draw_masks, without device row counts."""
    fps_w, fps_h = (0, 0) if fps_box is None else (int(fps_box[0]), int(fps_box[1]))
    if fps_w < 0 or fps_h < 0:
        raise ValueError("render: fps_box sizes must be >= 0, got %s" % ((fps_w, fps_h),))
    return _lib.YbRenderOpts(None, fps_w, fps_h, 1 if draw_masks else 0)


def _outputs(frames, top_k, dev):
    """The images and `drawn` tensors one render call writes, and an item per frame pointing at them."""
    B = len(frames)
    drawn = {"num": torch.zeros(B, dtype=torch.int32, device=dev),
             "classes": torch.zeros(B, top_k, dtype=torch.int64, device=dev),
             "scores": torch.zeros(B, top_k, dtype=torch.float32, device=dev),
             "boxes": torch.zeros(B, top_k, 4, dtype=torch.int64, device=dev)}
    images = [torch.empty(int(f.shape[0]), int(f.shape[1]), 3, dtype=torch.uint8, device=dev) for f in frames]
    items = (_lib.YbRenderItem * B)()
    num, classes, scores, boxes = drawn["num"], drawn["classes"], drawn["scores"], drawn["boxes"]
    for i, f in enumerate(frames):
        it = items[i]
        it.frame, it.out = f.data_ptr(), images[i].data_ptr()
        it.sel_n, it.sel_cls = num[i:].data_ptr(), classes[i].data_ptr()
        it.sel_score, it.sel_box = scores[i].data_ptr(), boxes[i].data_ptr()
        it.h, it.w = int(f.shape[0]), int(f.shape[1])
    return images, drawn, items


def _render(items, frames, dev, ph, pw, k, crop_masks, top_k, score_threshold, class_color, mask_alpha, opts):
    lib = _lib.load()
    _lib.check(lib.yb_render_list_ex(_ops_handle(dev, k), items, len(frames), 1 if frames[0].dtype == torch.uint8 else 0,
                                     ph, pw, k, 1 if crop_masks else 0, top_k, float(score_threshold),
                                     1 if class_color else 0, float(mask_alpha), _lib.ptr(_palette(dev)),
                                     len(_config.COLORS), ctypes.byref(opts), _lib.current_stream(dev)),
               "yb_render_list_ex")


def _on_device(det_output, dev):
    """det_output with every detection that is on another GPU than dev copied to dev (det_output is left as it is).
    The copy is torch's device-to-device copy: it runs on the detections' device's current stream, so it follows the
    network call that enqueued them there (DataParallel's replica k enqueues on cuda:k's current stream), and dev's
    current stream waits for it."""
    out = []
    for d in det_output:
        det = d['detection']
        if det is not None and det['box'].is_cuda and det['box'].device != dev:
            d = dict(d, detection={k: v.to(dev) for k, v in det.items()})
        out.append(d)
    return out


def render_masks(det_output, frames, top_k=5, score_threshold=0, class_color=False, mask_alpha=0.45, crop_masks=True,
                 fps_box=None, draw_masks=True):
    """frames: a list of CUDA [h_i,w_i,3] BGR tensors or one [B,h,w,3] tensor, uint8 or float32 0..255, one per entry of
    det_output (Yolact's output list).  fps_box: None or (text_w, text_h); draw_masks: blend the masks (see the module
    docstring).  Returns (images, drawn): images a list of CUDA uint8 [h_i,w_i,3]; drawn a dict of device tensors num,
    classes, scores, boxes (see the module docstring).  Detections on another GPU than the frames (a DataParallel
    replica's) are copied to the frames' device first, so the images are those of the same-device render, bit for
    bit."""
    frames = _frame_list(frames, "render_masks")
    if len(frames) != len(det_output):
        raise ValueError("render_masks: %d frames for %d detections" % (len(frames), len(det_output)))
    top_k = int(top_k)
    if top_k < 1:
        raise ValueError("render_masks: top_k must be >= 1")
    frames, dev = _checked_frames(frames, "render_masks")
    opts = _opts(fps_box, draw_masks)
    B = len(frames)
    images, drawn, items = _outputs(frames, top_k, dev)
    if B == 0:
        return [], drawn

    g = _gather(_on_device(det_output, dev), "render_masks")
    dets = dict(zip(g.live, g.dets))
    keep_alive = []   # the contiguous inputs, held until the call has enqueued its reads of them
    ph, pw, k = g.shape if g.eval_mask_branch else (1, 1, 4)
    rank = {i: d['score'] for i, d in dets.items()}
    if g.use_maskiou:
        # YOLACT++ (output_utils.py:77-88 with rescore_bbox, eval.py:148-149): maskiou_net on the prototype-resolution
        # masks of every row of every image at once; the rows are independent, so the score filter can follow
        pm = torch.empty(sum(g.ns), ph, pw, dtype=torch.float32, device=dev)
        _post_list(dev, [(d['proto'], d['mask'], d['box'], int(frames[i].shape[0]), int(frames[i].shape[1]))
                         for i, d in dets.items()], ph, pw, k, crop_masks, pm=pm)
        rescored = _rescore_list(g.net, g.ncfg, pm, [d['class'] for d in g.dets], [d['score'] for d in g.dets], g.ns)
        if rescored is not None:
            rank.update(zip(g.live, rescored[0]))

    for i in range(B):
        it = items[i]
        d = dets.get(i)
        n = int(d['box'].shape[0]) if d is not None else 0
        if n > 0:
            box = d['box'].contiguous().float()
            cls = d['class'].contiguous().long()
            det_score = d['score'].contiguous().float()
            score = rank[i].contiguous().float()
            keep_alive += [box, cls, det_score, score]
            it.box, it.cls, it.det_score, it.score = box.data_ptr(), cls.data_ptr(), det_score.data_ptr(), score.data_ptr()
            if g.eval_mask_branch:
                proto, coef = d['proto'].contiguous().float(), d['mask'].contiguous().float()
                keep_alive += [proto, coef]
                it.proto, it.coef = proto.data_ptr(), coef.data_ptr()
        it.n = n
    _render(items, frames, dev, ph, pw, k, crop_masks, top_k, score_threshold, class_color, mask_alpha, opts)
    return images, drawn


def render_frames(net, frames, top_k=5, score_threshold=0, class_color=False, mask_alpha=0.45, crop_masks=True,
                  fps_box=None, draw_masks=True):
    """render_masks(net.forward_frames(frames), frames, ...) bit for bit, images and `drawn` alike, with no host sync:
    net.infer_frames, then one yb_render_list_ex whose items point into the padded outputs (capacity M rows per image)
    and whose selection reads Detect's row counts on the device.  frames: CUDA uint8 [B,h,w,3] or a list of [h_i,w_i,3],
    as infer_frames takes them.  Yolact.render_frames is this with net = self."""
    if net.training:
        raise RuntimeError("Yolact.render_frames is the eval-mode path; call net.eval() first")
    top_k = int(top_k)
    if top_k < 1:
        raise ValueError("render_frames: top_k must be >= 1")
    opts = _opts(fps_box, draw_masks)   # refuses bad sizes before the network runs
    flist, dev = _checked_frames(_frame_list(frames, "render_frames"), "render_frames")
    if not flist:
        return render_masks([], [], top_k=top_k)
    out, oh, ow = net._infer_frames(frames if isinstance(frames, (list, tuple)) else frames.contiguous(), None)
    _config.cfg._tmp_img_h, _config.cfg._tmp_img_w = oh, ow   # as forward_frames sets them
    box, coef, cls, score, count, proto = out
    B, M = int(box.shape[0]), int(box.shape[1])
    k = int(coef.shape[2])
    opts.d_counts = count.data_ptr()
    images, drawn, items = _outputs(flist, top_k, dev)
    cfg = _config.cfg
    eval_mask_branch = getattr(cfg, "eval_mask_branch", True) and proto is not None
    ph, pw = (int(proto.shape[1]), int(proto.shape[2])) if eval_mask_branch else (1, 1)
    if not eval_mask_branch:
        k = 4
    rank = score
    ncfg = net.cfg
    if eval_mask_branch and bool(getattr(ncfg, "use_maskiou", False)) and M > 0:
        # YOLACT++: maskiou_net over all B*M padded rows at once (rows are independent and maskiou_net is bit-identical
        # whatever the batch, DESIGN.md section 3.3, so each real row ranks as on render_masks' list path).  The rows at
        # or past an image's count are whatever Detect left in the padded buffers: their box, coefficients and class
        # are zeroed here, so they crop to empty prototype masks and gather a valid class, and they cannot fault or
        # leak.  Their ranking scores are never read: the selection stops at the device count.
        valid = torch.arange(M, device=dev)[None, :] < count[:, None].long()
        zbox = torch.where(valid[..., None], box, 0.0)
        zcoef = torch.where(valid[..., None], coef, 0.0)
        zcls = torch.where(valid, cls, 0)
        pm = torch.empty(B * M, ph, pw, dtype=torch.float32, device=dev)
        _post_list(dev, [(proto[b], zcoef[b], zbox[b], int(flist[b].shape[0]), int(flist[b].shape[1]))
                         for b in range(B)], ph, pw, k, crop_masks, pm=pm)
        rescored = _rescore_list(net, ncfg, pm, [zcls.reshape(-1)], [score.reshape(-1)], [B * M])
        if rescored is not None:
            rank = rescored[0][0].reshape(B, M)
    for b in range(B):
        it = items[b]
        it.box, it.cls, it.det_score, it.score = (box[b].data_ptr(), cls[b].data_ptr(), score[b].data_ptr(),
                                                  rank[b].data_ptr())
        if eval_mask_branch:
            it.proto, it.coef = proto[b].data_ptr(), coef[b].data_ptr()
        it.n = M   # the capacity: the selection reads row count count[b] on the device
    _render(items, flist, dev, ph, pw, k, crop_masks, top_k, score_threshold, class_color, mask_alpha, opts)
    return images, drawn
