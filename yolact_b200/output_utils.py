"""postprocess: drop-in for layers/output_utils.py:15-122 (lincomb path) on the CUDA library.

    classes, scores, boxes, masks = postprocess(det_output, w, h, batch_idx=0,
                                                interpolation_mode='bilinear', visualize_lincomb=False,
                                                crop_masks=True, score_threshold=0)

Same argument meaning and return types as the reference: classes int64 [n], scores f32 [n] (or the
2-list [scores, scores*maskiou] for YOLACT++ unless cfg.rescore_bbox, output_utils.py:84-88), boxes
int64 [n,4] absolute pixels, masks f32 [n,h,w] in {0,1}; four empty tensors when there is nothing
(output_utils.py:39-40,49-50).  The whole mask pipeline (coef x proto -> sigmoid -> crop -> bilinear ->
> 0.5) is ONE kernel (yb_postprocess).

Differences (documented in INTEGRATION.md): the reference writes the sanitised absolute boxes back
into det_output['box'] in place (output_utils.py:97-98, SURVEY.md Appendix D.1); this function
leaves its input untouched.  `mask_format` ('f32' | 'u8' | 'bits') is an extension: 'bits' returns
uint32 words, 1 bit per pixel, row pitch ceil(w/32) -- 32x less HBM/PCIe traffic than fp32.

postprocess_list(det_output, sizes, ...) is postprocess for every image of a list at its own size (a folder of images
through Yolact.forward_frames), in one call with one launch per kernel for the whole list.
"""
import ctypes

import torch

from . import _lib
from . import config as _config

_FORMATS = {"f32": _lib.YB_MASK_F32, "u8": _lib.YB_MASK_U8, "bits": _lib.YB_MASK_BITS}
_ops_handles = {}


def _ops_handle(device, mask_dim=32):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    key = (idx, mask_dim)
    if key not in _ops_handles:
        lib = _lib.load()
        yc = _lib.YbConfig()
        yc.backbone = _lib.YB_BACKBONE_NONE
        yc.num_classes = 81
        yc.mask_dim = mask_dim
        yc.precision = _lib.YB_PREC_F32
        yc.nms_top_k, yc.nms_conf_thresh, yc.nms_thresh, yc.max_num_detections = 200, 0.05, 0.5, 100
        h = ctypes.c_void_p()
        _lib.check(lib.yb_create(ctypes.byref(yc), idx, ctypes.byref(h)), "yb_create(ops)")
        _ops_handles[key] = h
    return _ops_handles[key]


def launch_count():
    """Kernel launches issued by the postprocess ops handles (bench.py's gpu_launches)."""
    lib = _lib.load()
    return sum(int(lib.yb_launch_count(h)) for h in _ops_handles.values())


def assemble_masks(proto, coef, boxes, h, w, crop_masks=True, mask_format="f32", want_proto_masks=False,
                   masks_out=None):
    """Low-level: proto [ph,pw,k], coef [n,k], boxes [n,4] relative -> (masks, boxes_px int64 [n,4],
    proto_masks [n,ph,pw] or None).  No host sync."""
    if not proto.is_cuda:
        raise _lib.YbError("yolact_b200.postprocess runs on CUDA (H100) only; there is no CPU path.")
    lib = _lib.load()
    dev = proto.device
    n = int(coef.shape[0])
    ph, pw, k = (int(s) for s in proto.shape)
    proto = proto.contiguous().float()
    coef = coef.contiguous().float()
    boxes = boxes.contiguous().float()
    fmt = _FORMATS[mask_format]
    masks = masks_out if masks_out is not None else _empty_masks((n,), h, w, fmt, dev)
    boxes_px = torch.empty(n, 4, dtype=torch.int64, device=dev)
    pm = torch.empty(n, ph, pw, dtype=torch.float32, device=dev) if want_proto_masks else None
    if n > 0:
        _lib.check(lib.yb_postprocess(_ops_handle(dev, k), _lib.ptr(proto), ph, pw, k, _lib.ptr(coef), _lib.ptr(boxes),
                                      n, h, w, 1 if crop_masks else 0, fmt, _lib.ptr(masks), _lib.ptr(boxes_px),
                                      _lib.ptr(pm), _lib.current_stream(dev)), "yb_postprocess")
    return masks, boxes_px, pm


def assemble_masks_batch(proto, coef, boxes, h, w, crop_masks=True, mask_format="f32", masks_out=None,
                         boxes_out=None):
    """Whole batch in one launch: proto [B,ph,pw,k], coef [B,n,k], boxes [B,n,4] (padded rows, e.g.
    Yolact.infer_padded's outputs) -> (masks [B,n,...], boxes_px int64 [B,n,4]).  No host sync."""
    if not proto.is_cuda:
        raise _lib.YbError("yolact_b200.postprocess runs on CUDA (H100) only; there is no CPU path.")
    lib = _lib.load()
    dev = proto.device
    B, ph, pw, k = (int(s) for s in proto.shape)
    n = int(coef.shape[1])
    proto, coef, boxes = proto.contiguous().float(), coef.contiguous().float(), boxes.contiguous().float()
    fmt = _FORMATS[mask_format]
    masks = masks_out if masks_out is not None else _empty_masks((B, n), h, w, fmt, dev)
    boxes_px = boxes_out if boxes_out is not None else torch.empty(B, n, 4, dtype=torch.int64, device=dev)
    if n > 0 and B > 0:
        _lib.check(lib.yb_postprocess_batch(_ops_handle(dev, k), _lib.ptr(proto), ph, pw, k, _lib.ptr(coef),
                                            _lib.ptr(boxes), n, B, h, w, 1 if crop_masks else 0, fmt, _lib.ptr(masks),
                                            _lib.ptr(boxes_px), _lib.current_stream(dev)), "yb_postprocess_batch")
    return masks, boxes_px


def postprocess(det_output, w, h, batch_idx=0, interpolation_mode='bilinear', visualize_lincomb=False,
                crop_masks=True, score_threshold=0, mask_format="f32"):
    cfg = _config.cfg
    dets = det_output[batch_idx]
    net = dets['net']
    dets = dets['detection']
    if dets is None:
        return [torch.Tensor()] * 4  # output_utils.py:39-40

    if score_threshold > 0:
        keep = dets['score'] > score_threshold
        for k in dets:
            if k != 'proto':
                dets[k] = dets[k][keep]
        if dets['score'].size(0) == 0:
            return [torch.Tensor()] * 4

    classes, boxes, scores, masks = dets['class'], dets['box'], dets['score'], dets['mask']
    ncfg = getattr(net, "cfg", cfg)
    eval_mask_branch = getattr(cfg, "eval_mask_branch", True) and 'proto' in dets

    if eval_mask_branch:
        if interpolation_mode != 'bilinear':
            raise NotImplementedError("yolact_b200.postprocess implements bilinear upsampling only "
                                      "(the only mode eval.py uses)")
        if visualize_lincomb:
            raise NotImplementedError("display_lincomb (debug visualisation) is out of scope")
        use_maskiou = bool(getattr(ncfg, "use_maskiou", False))
        out_masks, boxes_px, pm = assemble_masks(dets['proto'], masks, boxes, h, w, crop_masks, mask_format,
                                                 want_proto_masks=use_maskiou)
        if use_maskiou:
            rescored = _maskiou_rescore(net, ncfg, pm, classes, scores)
            if rescored is not None:
                scores = rescored[0] if rescored[1] else [scores, rescored[0]]
        masks = out_masks
    else:
        # cfg.eval_mask_branch == False (--detect): boxes only, masks are the raw coefficients (Appendix D.15)
        boxes_px = _boxes_only(boxes, h, w)

    return classes, scores, boxes_px, masks


def postprocess_list(det_output, sizes, interpolation_mode='bilinear', visualize_lincomb=False, crop_masks=True,
                     score_threshold=0, mask_format="f32"):
    """postprocess for every image of det_output at its own size, in one call:
    [postprocess(det_output, w_i, h_i, i, ...) for i, (h_i, w_i) in enumerate(sizes)], bit for bit, and det_output is
    left as those calls leave it.  sizes[i] = (h_i, w_i), i.e. frame i's shape[:2] -- what Yolact.forward_frames' list
    of differently sized frames needs back.

    One yb_postprocess_list call covers the whole list (boxes and masks, plus the prototype-resolution masks of
    YOLACT++), and YOLACT++ runs maskiou_net once over the rows of all images, so the launches do not grow with the
    list.  With score_threshold == 0 there is no host sync; with score_threshold > 0 there is one, for the kept-row
    counts of all images together.  The threshold keeps each image's leading rows (Detect's scores are descending):
    rows that are not a prefix raise ValueError rather than silently differ from postprocess."""
    if len(sizes) != len(det_output):
        raise ValueError("postprocess_list: %d sizes for %d images" % (len(sizes), len(det_output)))
    hw = []
    for s in sizes:
        h, w = (int(v) for v in s)
        if h <= 0 or w <= 0:
            raise ValueError("postprocess_list: image sizes must be positive, got %s" % (tuple(s),))
        hw.append((h, w))
    empty = [torch.Tensor()] * 4   # output_utils.py:39-40,49-50
    live = [i for i, d in enumerate(det_output) if d['detection'] is not None]
    for i in live:
        if not det_output[i]['detection']['box'].is_cuda:
            raise _lib.YbError("yolact_b200.postprocess runs on CUDA (H100) only; there is no CPU path.")
    dev = det_output[live[0]]['detection']['box'].device if live else None

    if score_threshold > 0 and live:
        _keep_leading_rows(det_output, live, score_threshold, dev)
        live = [i for i in live if det_output[i]['detection']['score'].size(0) > 0]
    out = [empty] * len(det_output)
    if not live:
        return out

    cfg = _config.cfg
    dets = [det_output[i]['detection'] for i in live]
    with_proto = ['proto' in d for d in dets]
    if any(with_proto) and not all(with_proto):
        raise ValueError("postprocess_list: some detections carry 'proto' and some do not")
    eval_mask_branch = getattr(cfg, "eval_mask_branch", True) and with_proto[0]
    lib = _lib.load()
    stream = _lib.current_stream(dev)
    ns = [int(d['box'].shape[0]) for d in dets]
    keep_alive = []   # the contiguous inputs, held until the call has enqueued its reads of them
    items = (_lib.YbPostItem * len(dets))()

    if not eval_mask_branch:
        # cfg.eval_mask_branch == False (--detect): boxes only, masks are the raw coefficients (Appendix D.15)
        dummy = torch.empty(4, dtype=torch.float32, device=dev)   # never read without masks
        for j, (i, d, n) in enumerate(zip(live, dets, ns)):
            box = d['box'].contiguous().float()
            boxes_px = torch.empty(n, 4, dtype=torch.int64, device=dev)
            keep_alive.append(box)
            items[j] = _lib.YbPostItem(dummy.data_ptr(), dummy.data_ptr(), box.data_ptr(), None, boxes_px.data_ptr(),
                                       None, n, hw[i][0], hw[i][1])
            out[i] = (d['class'], d['score'], boxes_px, d['mask'])
        _lib.check(lib.yb_postprocess_list(_ops_handle(dev, 4), items, len(dets), 1, 1, 4, 0, _lib.YB_MASK_F32, stream),
                   "yb_postprocess_list(boxes)")
        return out

    if interpolation_mode != 'bilinear':
        raise NotImplementedError("yolact_b200.postprocess implements bilinear upsampling only "
                                  "(the only mode eval.py uses)")
    if visualize_lincomb:
        raise NotImplementedError("display_lincomb (debug visualisation) is out of scope")
    shapes = {tuple(int(s) for s in d['proto'].shape) for d in dets}
    if len(shapes) != 1:
        raise ValueError("postprocess_list: the images' prototypes differ in (ph, pw, k): %s" % sorted(shapes))
    ph, pw, k = shapes.pop()
    net = det_output[live[0]]['net']
    ncfg = getattr(net, "cfg", cfg)
    use_maskiou = bool(getattr(ncfg, "use_maskiou", False))
    if use_maskiou and any(det_output[i]['net'] is not net for i in live):
        raise ValueError("postprocess_list: maskiou rescoring needs every image to come from the same net")
    fmt = _FORMATS[mask_format]
    pm = torch.empty(sum(ns), ph, pw, dtype=torch.float32, device=dev) if use_maskiou else None
    off = 0
    for j, (i, d, n) in enumerate(zip(live, dets, ns)):
        h, w = hw[i]
        proto, coef, box = d['proto'].contiguous().float(), d['mask'].contiguous().float(), d['box'].contiguous().float()
        masks = _empty_masks((n,), h, w, fmt, dev)
        boxes_px = torch.empty(n, 4, dtype=torch.int64, device=dev)
        keep_alive += [proto, coef, box]
        items[j] = _lib.YbPostItem(proto.data_ptr(), coef.data_ptr(), box.data_ptr(), masks.data_ptr() or None,
                                   boxes_px.data_ptr() or None, pm[off:off + n].data_ptr() if use_maskiou else None,
                                   n, h, w)
        out[i] = (d['class'], d['score'], boxes_px, masks)
        off += n
    _lib.check(lib.yb_postprocess_list(_ops_handle(dev, k), items, len(dets), ph, pw, k, 1 if crop_masks else 0, fmt,
                                       stream), "yb_postprocess_list")

    if use_maskiou and off > 0:
        # maskiou_net and the gather are per row: one call over the rows of every image at once
        cat = (lambda ts: torch.cat(ts)) if len(dets) > 1 else (lambda ts: ts[0])
        rescored = _maskiou_rescore(net, ncfg, pm, cat([d['class'] for d in dets]), cat([d['score'] for d in dets]))
        if rescored is not None:
            off = 0
            for i, d, n in zip(live, dets, ns):
                r = rescored[0][off:off + n]
                out[i] = (d['class'], r if rescored[1] else [d['score'], r]) + out[i][2:]
                off += n
    return out


def _empty_masks(lead, h, w, fmt, dev):
    """Uninitialised masks [*lead, h, w] in yb_mask_format fmt: fp32, uint8, or int32 words of 32 pixels per row."""
    if fmt == _lib.YB_MASK_F32:
        return torch.empty(*lead, h, w, dtype=torch.float32, device=dev)
    if fmt == _lib.YB_MASK_U8:
        return torch.empty(*lead, h, w, dtype=torch.uint8, device=dev)
    return torch.empty(*lead, h, (w + 31) // 32, dtype=torch.int32, device=dev)


def _maskiou_rescore(net, ncfg, pm, classes, scores):
    """output_utils.py:79-88: maskiou_net on the cropped prototype-resolution masks pm [n,ph,pw], gathered at each row's
    class.  None unless cfg.rescore_mask; else (scores * maskiou, rescore_bbox): with rescore_bbox the rescored scores
    replace the scores, without it the reference returns [scores, scores * maskiou]."""
    lib = _lib.load()
    n, ph, pw = (int(s) for s in pm.shape)
    miou = torch.empty(n, dtype=torch.float32, device=pm.device)
    _lib.check(lib.yb_maskiou(net._handle_for(pm.device), _lib.ptr(pm), n, ph, pw, _lib.ptr(classes.contiguous().long()),
                              _lib.ptr(miou), _lib.current_stream(pm.device)), "yb_maskiou")
    if not getattr(ncfg, "rescore_mask", False):
        return None
    return scores * miou, getattr(_config.cfg, "rescore_bbox", False) or getattr(ncfg, "rescore_bbox", False)


def _keep_leading_rows(det_output, live, score_threshold, dev):
    """postprocess's `dets[k] = dets[k][dets['score'] > score_threshold]` for every live image, with ONE host sync:
    the kept-row counts of all images are computed together, and each image keeps that many leading rows.  Raises
    ValueError (before changing anything) when an image's kept rows are not its leading rows."""
    scores = [det_output[i]['detection']['score'] for i in live]
    lens = [int(s.shape[0]) for s in scores]
    flat = torch.cat(scores) if len(scores) > 1 else scores[0]
    keep = flat > score_threshold
    # image index and row index of every row, built on the host from the shapes and uploaded without a sync
    seg_pos = torch.stack([torch.repeat_interleave(torch.arange(len(lens)), torch.tensor(lens)),
                           torch.cat([torch.arange(n) for n in lens])]).to(dev, non_blocking=True)
    seg, pos = seg_pos[0], seg_pos[1]
    counts = torch.zeros(len(lens), dtype=torch.int64, device=dev).index_add_(0, seg, keep.long())
    stray = torch.zeros(len(lens), dtype=torch.int64, device=dev).index_add_(0, seg, (keep != (pos < counts[seg])).long())
    counts, stray = torch.stack([counts, stray]).tolist()   # the one host sync
    for i, n, bad in zip(live, counts, stray):
        if bad:
            raise ValueError("postprocess_list: score_threshold keeps rows of image %d that are not its leading rows "
                             "(its scores are not in descending order); run postprocess on it" % i)
    for i, n in zip(live, counts):
        dets = det_output[i]['detection']
        for k in dets:
            if k != 'proto':
                dets[k] = dets[k][:n]


def _boxes_only(boxes, h, w):
    """boxes [n,4] relative -> int64 [n,4] pixels: yb_postprocess without masks (its proto and coef are never read)."""
    lib = _lib.load()
    dev = boxes.device
    n = int(boxes.shape[0])
    boxes = boxes.contiguous().float()
    boxes_px = torch.empty(n, 4, dtype=torch.int64, device=dev)
    dummy = torch.zeros(4, device=dev)
    _lib.check(lib.yb_postprocess(_ops_handle(dev, 4), _lib.ptr(dummy), 1, 1, 4, _lib.ptr(dummy), _lib.ptr(boxes), n, h,
                                  w, 0, _lib.YB_MASK_F32, None, _lib.ptr(boxes_px), None, _lib.current_stream(dev)),
               "yb_postprocess(boxes)")
    return boxes_px


def unpack_bits(words, w):
    """[n,h,ceil(w/32)] int32 bit masks -> [n,h,w] uint8 (host/torch helper for consumers)."""
    n, h, wp = words.shape
    shifts = torch.arange(32, device=words.device, dtype=torch.int32)
    bits = (words.unsqueeze(-1) >> shifts) & 1
    return bits.reshape(n, h, wp * 32)[:, :, :w].to(torch.uint8)
