"""dcn_v2: op-level drop-in for external/DCNv2/dcn_v2.py (forward only, inference).

`dcn_v2_conv(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups)` and the
`DCN` / `DCNv2` modules keep the reference's names and argument order (dcn_v2.py:16-128); the
computation is yb_dcn_forward (the C-ABI mirror of dcn_v2_forward, src/dcn_v2.h:9-23).  The
reference's extension cannot be built against modern PyTorch (THC headers); this one needs no
torch C++ API at all.  Backward is not implemented (training is out of scope).
"""
import ctypes
import math

import torch
from torch import nn
from torch.nn.modules.utils import _pair

from . import _lib

_handles = {}


def _handle(device, precision):
    idx = device.index if device.index is not None else torch.cuda.current_device()
    key = (idx, precision)
    if key not in _handles:
        lib = _lib.load()
        yc = _lib.YbConfig()
        yc.backbone = _lib.YB_BACKBONE_NONE
        yc.num_classes, yc.mask_dim = 81, 32
        yc.precision = precision
        yc.nms_top_k, yc.nms_conf_thresh, yc.nms_thresh, yc.max_num_detections = 200, 0.05, 0.5, 100
        h = ctypes.c_void_p()
        _lib.check(lib.yb_create(ctypes.byref(yc), idx, ctypes.byref(h)), "yb_create(ops)")
        _handles[key] = h
    return _handles[key]


def dcn_v2_conv(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups, precision="f32"):
    if not input.is_cuda:
        raise _lib.YbError("yolact_b200.dcn_v2 runs on CUDA (H100) only (the reference's CPU path is an AT_ERROR stub too)")
    lib = _lib.load()
    sh, sw = _pair(stride)
    ph, pw = _pair(padding)
    dh, dw = _pair(dilation)
    B, C, H, W = input.shape
    Co, _, kh, kw = weight.shape
    Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    out = torch.empty(B, Co, Ho, Wo, device=input.device, dtype=torch.float32)
    args = [t.contiguous().float() for t in (input, weight, bias, offset, mask)]
    prec = _lib.PRECISIONS[precision]
    _lib.check(lib.yb_dcn_forward(_handle(input.device, prec), _lib.ptr(args[0]), _lib.ptr(args[1]), _lib.ptr(args[2]),
                                  _lib.ptr(args[3]), _lib.ptr(args[4]), _lib.ptr(out), B, C, H, W, Co, kh, kw, sh, sw,
                                  ph, pw, dh, dw, deformable_groups, _lib.current_stream(input.device)),
               "yb_dcn_forward")
    return out


class DCNv2(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.deformable_groups = deformable_groups
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels, *self.kernel_size))
        self.bias = nn.Parameter(torch.Tensor(out_channels))
        n = in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)
        self.bias.data.zero_()

    def forward(self, input, offset, mask):
        assert 2 * self.deformable_groups * self.kernel_size[0] * self.kernel_size[1] == offset.shape[1]
        assert self.deformable_groups * self.kernel_size[0] * self.kernel_size[1] == mask.shape[1]
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)


class DCN(DCNv2):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, deformable_groups)
        channels_ = self.deformable_groups * 3 * self.kernel_size[0] * self.kernel_size[1]
        self.conv_offset_mask = nn.Conv2d(self.in_channels, channels_, kernel_size=self.kernel_size,
                                          stride=self.stride, padding=self.padding, bias=True)
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, input):
        # dcn_v2.py:118-128: the offset/mask conv is a plain conv (cuDNN in the reference, library call here
        # only in this standalone module; inside Yolact it runs on our own kernels)
        out = self.conv_offset_mask(input)
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        mask = torch.sigmoid(mask)
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)
