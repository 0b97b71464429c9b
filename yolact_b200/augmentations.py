"""FastBaseTransform: drop-in for utils/augmentations.py:616-658 on the CUDA library.

    transform = FastBaseTransform()
    batch = transform(frame.unsqueeze(0))        # frame: [h,w,3] BGR, uint8 or float (0..255), on the GPU
    preds = net(batch)

One kernel: HWC BGR -> bilinear resize (F.interpolate, align_corners=False) -> normalise -> RGB ->
NCHW fp32.  uint8 frames are accepted directly (the reference needs `.float()` first: 4x the H2D bytes).
Like the reference, only channel_order == 'RGB' is supported, and cfg.preserve_aspect_ratio follows
Resize.calc_size_preserve_ar (utils/augmentations.py:129-138).
"""
import ctypes
from math import sqrt

import torch

from . import _lib
from . import config as _config
from .output_utils import _ops_handle


def calc_size_preserve_ar(img_w, img_h, max_size):
    """Resize.calc_size_preserve_ar (utils/augmentations.py:129-138): keep the area at max_size^2."""
    ratio = sqrt(img_w / img_h)
    w = max_size * ratio
    h = max_size / ratio
    return int(w), int(h)


class FastBaseTransform(torch.nn.Module):
    def __init__(self, cfg=None):
        super().__init__()
        self.cfg = cfg if cfg is not None else _config.cfg
        self.mean = _config.MEANS
        self.std = _config.STD

    def _mode(self):
        c = self.cfg
        if getattr(c, "normalize", True):
            return _lib.YB_XFORM_NORMALIZE
        if getattr(c, "subtract_means", False):
            return _lib.YB_XFORM_SUBTRACT_MEANS
        if getattr(c, "to_float", False):
            return _lib.YB_XFORM_TO_FLOAT
        return _lib.YB_XFORM_NONE

    def forward(self, img):
        if not img.is_cuda:
            raise _lib.YbError("yolact_b200.FastBaseTransform runs on CUDA (H100) only; there is no CPU path.")
        if getattr(self.cfg, "channel_order", "RGB") != "RGB":
            raise NotImplementedError   # utils/augmentations.py:648-649
        B, H, W, C = (int(s) for s in img.shape)
        if C != 3:
            raise ValueError("FastBaseTransform expects [n, h, w, 3] BGR frames")
        S = int(self.cfg.max_size)
        if getattr(self.cfg, "preserve_aspect_ratio", False):
            ow, oh = calc_size_preserve_ar(W, H, S)
        else:
            oh = ow = S
        is_u8 = img.dtype == torch.uint8
        x = img.contiguous() if is_u8 else img.contiguous().float()
        out = torch.empty(B, 3, oh, ow, dtype=torch.float32, device=img.device)
        mean = (ctypes.c_float * 3)(*self.mean)
        std = (ctypes.c_float * 3)(*self.std)
        lib = _lib.load()
        _lib.check(lib.yb_fast_base_transform(_ops_handle(img.device), _lib.ptr(x), 1 if is_u8 else 0, B, H, W, oh, ow,
                                              self._mode(), mean, std, _lib.ptr(out), _lib.current_stream(img.device)),
                   "yb_fast_base_transform")
        return out
