"""eval.py-side consumers of the path's results, on the CUDA library (SURVEY.md section 8f row 2).

    mask_iou(masks_a, masks_b, iscrowd=False)      <- layers/box_utils.py:98-113  (eval.py:435 _mask_iou)
    jaccard(box_a, box_b, iscrowd=False)           <- layers/box_utils.py:54-79   (eval.py:442 _bbox_iou)
    encode_masks(masks)                            <- pycocotools.mask.encode in Detections.add_mask (eval.py:320-330)
    display_blend(img, masks, colors, alpha)       <- the GPU mask blend inside prep_display (eval.py:186-209,226)
    get_color(j, classes, class_color)             <- prep_display's palette lookup (eval.py:169-183)

prep_display itself (eval.py:135-262) is caller code and is NOT rebuilt here: a caller that keeps its own loop replaces
the ten ATen ops of the blend by `display_blend`; yolact_b200.display.render_masks does the whole GPU part (postprocess
to .byte()) for a list of frames and leaves only the OpenCV text and boxes to the caller (INTEGRATION.md section 1).

The reference multiplies two dense float matrices for the mask IoU and ships fp32 masks over PCIe for the RLE;
here masks are 1 bit per pixel on the GPU (32x fewer bytes), the IoU is AND + popcount, and only the run
lengths (a few KB per image) cross PCIe.  mask_iou is bit-identical to the reference (integer counts, one
fp32 division); the RLE string is the one pycocotools produces (maskApi.c rleToString), built on the host from
the GPU's run lengths.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from . import config as _config
from .output_utils import _FORMATS, _ops_handle, postprocess


def _require_cuda(t, what):
    if not t.is_cuda:
        raise _lib.YbError("yolact_b200.%s runs on CUDA (H100) only; there is no CPU path." % what)


def pack_masks(masks):
    """0/1 masks [n, ...] (float or uint8) -> int32 words [n, ceil(L/32)], L = prod of the trailing dims:
    the whole mask is one bit row, which is all mask_iou needs."""
    _require_cuda(masks, "pack_masks")
    n = int(masks.shape[0])
    flat = masks.reshape(n, -1)
    L = int(flat.shape[1])
    if flat.dtype == torch.uint8 or flat.dtype == torch.bool:
        flat, fmt = flat.contiguous().view(torch.uint8), _lib.YB_MASK_U8
    else:
        flat, fmt = flat.contiguous().float(), _lib.YB_MASK_F32
    bits = torch.empty(n, (L + 31) // 32, dtype=torch.int32, device=masks.device)
    if n > 0 and L > 0:
        lib = _lib.load()
        _lib.check(lib.yb_pack_mask_bits(_ops_handle(masks.device), _lib.ptr(flat), fmt, n, L, _lib.ptr(bits),
                                         _lib.current_stream(masks.device)), "yb_pack_mask_bits")
    return bits


def mask_iou(masks_a, masks_b, iscrowd=False, packed=False):
    """[a, h, w] x [b, h, w] (or the [a, h*w] views eval.py passes) -> [a, b] float32.
    packed=True: both inputs are already bit-packed int32 words with identical row pitch."""
    _require_cuda(masks_a, "mask_iou")
    a = masks_a if packed else pack_masks(masks_a)
    b = masks_b if packed else pack_masks(masks_b)
    if a.shape[1:] != b.shape[1:]:
        raise ValueError("mask_iou: the two mask sets have different sizes")
    a = a.reshape(a.shape[0], -1).contiguous()
    b = b.reshape(b.shape[0], -1).contiguous()
    n, m, words = int(a.shape[0]), int(b.shape[0]), int(a.shape[1])
    out = torch.empty(n, m, dtype=torch.float32, device=a.device)
    if n and m:
        lib = _lib.load()
        _lib.check(lib.yb_mask_iou(_ops_handle(a.device), _lib.ptr(a), n, _lib.ptr(b), m, words, 1 if iscrowd else 0,
                                   _lib.ptr(out), _lib.current_stream(a.device)), "yb_mask_iou")
    return out


def jaccard(box_a, box_b, iscrowd=False):
    """box_utils.py:54-79 for [A,4] x [B,4] (or batched [n,A,4] x [n,B,4])."""
    _require_cuda(box_a, "jaccard")
    if box_a.dim() == 3:
        return torch.stack([jaccard(x, y, iscrowd) for x, y in zip(box_a, box_b)])
    a, b = box_a.contiguous().float(), box_b.contiguous().float()
    n, m = int(a.shape[0]), int(b.shape[0])
    out = torch.empty(n, m, dtype=torch.float32, device=a.device)
    if n and m:
        lib = _lib.load()
        _lib.check(lib.yb_box_iou(_ops_handle(a.device), _lib.ptr(a), n, _lib.ptr(b), m, 1 if iscrowd else 0,
                                  _lib.ptr(out), _lib.current_stream(a.device)), "yb_box_iou")
    return out


# ---- COCO RLE ----------------------------------------------------------------------------------------------
def mask_run_lengths(masks, mask_format=None, w=None, cap=None):
    """masks [n,h,w] (float / uint8) or bit-packed [n,h,ceil(w/32)] int32 with `w` given ->
    list of n uint32 numpy arrays: pycocotools' rleEncode `cnts` (column-major runs, zeros first)."""
    _require_cuda(masks, "mask_run_lengths")
    n, h = int(masks.shape[0]), int(masks.shape[1])
    if mask_format is None:
        mask_format = "bits" if masks.dtype == torch.int32 else ("u8" if masks.dtype in (torch.uint8, torch.bool) else "f32")
    if mask_format == "bits":
        if w is None:
            raise ValueError("bit-packed masks need the width `w`")
        m = masks.contiguous()
    else:
        w = int(masks.shape[2])
        m = masks.contiguous().view(torch.uint8) if mask_format == "u8" else masks.contiguous().float()
    if n == 0:
        return []
    lib = _lib.load()
    dev = masks.device
    cap = int(cap) if cap else min(h * w + 1, 4 * w + 64)
    while True:
        counts = torch.empty(n, cap, dtype=torch.int32, device=dev)
        nruns = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(lib.yb_mask_rle(_ops_handle(dev), _lib.ptr(m), _FORMATS[mask_format], n, h, int(w), _lib.ptr(counts),
                                   cap, _lib.ptr(nruns), _lib.current_stream(dev)), "yb_mask_rle")
        nr = nruns.cpu().numpy()
        if (nr > 0).all():
            break
        cap = int(-nr.min())   # some mask needed more room: one retry with the exact maximum
    host = counts[:, :int(nr.max())].cpu().numpy().view(np.uint32)
    return [host[i, :nr[i]].copy() for i in range(n)]


def rle_to_string(counts):
    """maskApi.c rleToString, vectorised: 5 data bits per character, continuation bit 0x20, values from
    the 4th on are deltas against counts[i-2]."""
    x = np.asarray(counts, np.int64).copy()
    if x.size > 3:
        x[3:] -= np.asarray(counts, np.int64)[1:-2]
    chars = np.zeros((x.size, 13), np.uint8)
    valid = np.zeros((x.size, 13), bool)
    live = np.ones(x.size, bool)
    for k in range(13):
        c = x & 0x1f
        x = x >> 5
        more = np.where((c & 0x10) != 0, x != -1, x != 0)
        chars[:, k] = (c | np.where(more, 0x20, 0)) + 48
        valid[:, k] = live
        live = live & more
        if not live.any():
            break
    return chars[valid].tobytes()


def encode_masks(masks, mask_format=None, w=None):
    """-> list of {'size': [h, w], 'counts': bytes}: what pycocotools.mask.encode(np.asfortranarray(m)) returns
    for each mask (eval.py:322)."""
    h = int(masks.shape[1])
    runs = mask_run_lengths(masks, mask_format, w)
    if w is None:
        w = int(masks.shape[2])
    return [{"size": [h, int(w)], "counts": rle_to_string(r)} for r in runs]


# ---- the mask blend of prep_display ------------------------------------------------------------------------
def get_color(j, classes, class_color=False, bgr=True):
    """eval.py:169-183: colour of the j-th drawn detection, as 0..255 ints (BGR like the frame unless bgr=False)."""
    colors = _config.COLORS
    idx = (int(classes[j]) * 5 if class_color else j * 5) % len(colors)
    c = colors[idx]
    return (c[2], c[1], c[0]) if bgr else c


def display_blend(img, masks, colors, mask_alpha=0.45, img_is_255=True, mask_format=None, w=None):
    """img [h,w,3] float on the GPU, masks [n,h,w] in drawing order, colors [n,3] 0..1 -> uint8 [h,w,3] (GPU)."""
    _require_cuda(img, "display_blend")
    h, wi = int(img.shape[0]), int(img.shape[1])
    n = int(masks.shape[0]) if masks is not None else 0
    if mask_format is None and n:
        mask_format = "bits" if masks.dtype == torch.int32 else ("u8" if masks.dtype in (torch.uint8, torch.bool) else "f32")
    fmt = _FORMATS[mask_format] if n else _lib.YB_MASK_F32
    if n:
        m = masks.contiguous() if mask_format == "bits" else (
            masks.contiguous().view(torch.uint8) if mask_format == "u8" else masks.contiguous().float())
        col = torch.as_tensor(colors, dtype=torch.float32, device=img.device).contiguous()
    else:
        m, col = None, None
    out = torch.empty(h, wi, 3, dtype=torch.uint8, device=img.device)
    x = img.contiguous().float()
    lib = _lib.load()
    _lib.check(lib.yb_display_blend(_ops_handle(img.device), _lib.ptr(x), 1 if img_is_255 else 0, _lib.ptr(m), fmt, n, h,
                                    wi, _lib.ptr(col), float(mask_alpha), _lib.ptr(out), _lib.current_stream(img.device)),
               "yb_display_blend")
    return out
