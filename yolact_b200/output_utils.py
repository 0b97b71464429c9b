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
    if masks_out is not None:
        masks = masks_out
    elif fmt == _lib.YB_MASK_F32:
        masks = torch.empty(n, h, w, dtype=torch.float32, device=dev)
    elif fmt == _lib.YB_MASK_U8:
        masks = torch.empty(n, h, w, dtype=torch.uint8, device=dev)
    else:
        masks = torch.empty(n, h, (w + 31) // 32, dtype=torch.int32, device=dev)
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
    if masks_out is not None:
        masks = masks_out
    elif fmt == _lib.YB_MASK_F32:
        masks = torch.empty(B, n, h, w, dtype=torch.float32, device=dev)
    elif fmt == _lib.YB_MASK_U8:
        masks = torch.empty(B, n, h, w, dtype=torch.uint8, device=dev)
    else:
        masks = torch.empty(B, n, h, (w + 31) // 32, dtype=torch.int32, device=dev)
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
            # output_utils.py:79-88: maskiou on the cropped prototype-resolution masks, gathered at class
            lib = _lib.load()
            n, ph, pw = pm.shape
            miou = torch.empty(n, dtype=torch.float32, device=pm.device)
            cls64 = classes.contiguous().long()
            _lib.check(lib.yb_maskiou(net._handle_for(pm.device), _lib.ptr(pm), int(n), int(ph), int(pw),
                                      _lib.ptr(cls64), _lib.ptr(miou), _lib.current_stream(pm.device)), "yb_maskiou")
            if getattr(ncfg, "rescore_mask", False):
                if getattr(cfg, "rescore_bbox", False) or getattr(ncfg, "rescore_bbox", False):
                    scores = scores * miou
                else:
                    scores = [scores, scores * miou]
        masks = out_masks
    else:
        # cfg.eval_mask_branch == False (--detect): boxes only, masks are the raw coefficients (Appendix D.15)
        _, boxes_px, _ = _boxes_only(boxes, h, w)

    return classes, scores, boxes_px, masks


def _boxes_only(boxes, h, w):
    lib = _lib.load()
    dev = boxes.device
    n = int(boxes.shape[0])
    boxes = boxes.contiguous().float()
    boxes_px = torch.empty(n, 4, dtype=torch.int64, device=dev)
    dummy = torch.zeros(1, 1, 4, device=dev)
    coef = torch.zeros(max(n, 1), 4, device=dev)
    if n > 0:
        _lib.check(lib.yb_postprocess(_ops_handle(dev, 4), _lib.ptr(dummy), 1, 1, 4, _lib.ptr(coef), _lib.ptr(boxes), n,
                                      h, w, 0, _lib.YB_MASK_F32, None, _lib.ptr(boxes_px), None,
                                      _lib.current_stream(dev)), "yb_postprocess(boxes)")
    return None, boxes_px, None


def unpack_bits(words, w):
    """[n,h,ceil(w/32)] int32 bit masks -> [n,h,w] uint8 (host/torch helper for consumers)."""
    n, h, wp = words.shape
    shifts = torch.arange(32, device=words.device, dtype=torch.int32)
    bits = (words.unsqueeze(-1) >> shifts) & 1
    return bits.reshape(n, h, wp * 32)[:, :, :w].to(torch.uint8)
