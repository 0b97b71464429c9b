"""dcn_v2: op-level drop-in for external/DCNv2/dcn_v2.py (forward only, inference).

`dcn_v2_conv(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups)` and the
`DCN` / `DCNv2` modules keep the reference's names and argument order (dcn_v2.py:16-128); the
computation is yb_dcn_forward_ex (the C-ABI mirror of dcn_v2_forward, src/dcn_v2.h:9-23): any kernel size,
per-axis stride / padding / dilation and deformable groups.  `dcn_v2_pooling(...)` and the `DCNv2Pooling` /
`DCNPooling` modules (dcn_v2.py:132-303) run yb_dcn_psroi_pool (dcn_v2_psroi_pooling_forward).  The
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
    geom = _lib.YbDcnParams(kh, kw, sh, sw, ph, pw, dh, dw, deformable_groups)
    _lib.check(lib.yb_dcn_forward_ex(_handle(input.device, prec), _lib.ptr(args[0]), _lib.ptr(args[1]),
                                     _lib.ptr(args[2]), _lib.ptr(args[3]), _lib.ptr(args[4]), _lib.ptr(out), B, C, H, W,
                                     Co, ctypes.byref(geom), _lib.current_stream(input.device)),
               "yb_dcn_forward_ex")
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


def dcn_v2_pooling(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                   sample_per_part=4, trans_std=.0):
    """Deformable PS-RoI pooling, forward (the reference's _DCNv2Pooling.apply, dcn_v2.py:132-184): input [N,C,H,W]
    with C = output_dim * group_size^2, rois [R,5] (batch index, x1, y1, x2, y2), offset [R, 2*num_classes, part, part]
    (unused when no_trans) -> [R, output_dim, pooled_size, pooled_size] fp32."""
    if not input.is_cuda:
        raise _lib.YbError("yolact_b200.dcn_v2 runs on CUDA (H100) only (the reference's CPU path is an AT_ERROR stub too)")
    lib = _lib.load()
    part_size = pooled_size if part_size is None else part_size
    no_trans = int(no_trans)
    N, C, H, W = input.shape
    R = rois.shape[0]
    x = input.contiguous().float()
    r = rois.contiguous().float()
    trans = None if no_trans else offset.contiguous().float()
    num_classes = 1 if no_trans else trans.shape[1] // 2
    out = torch.empty(R, output_dim, pooled_size, pooled_size, device=input.device, dtype=torch.float32)
    _lib.check(lib.yb_dcn_psroi_pool(_handle(input.device, _lib.YB_PREC_F32), _lib.ptr(x), _lib.ptr(r), _lib.ptr(trans),
                                     _lib.ptr(out), None, N, C, H, W, R, no_trans, num_classes, spatial_scale,
                                     output_dim, group_size, pooled_size, part_size, sample_per_part, trans_std,
                                     _lib.current_stream(input.device)),
               "yb_dcn_psroi_pool")
    return out


class DCNv2Pooling(nn.Module):
    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
        super().__init__()
        self.spatial_scale = spatial_scale
        self.pooled_size = pooled_size
        self.output_dim = output_dim
        self.no_trans = no_trans
        self.group_size = group_size
        self.part_size = pooled_size if part_size is None else part_size
        self.sample_per_part = sample_per_part
        self.trans_std = trans_std

    def forward(self, input, rois, offset):
        assert input.shape[1] == self.output_dim
        if self.no_trans:
            offset = input.new()
        return dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim, self.no_trans,
                              self.group_size, self.part_size, self.sample_per_part, self.trans_std)


class DCNPooling(DCNv2Pooling):
    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0, deform_fc_dim=1024):
        super().__init__(spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size, sample_per_part,
                         trans_std)
        self.deform_fc_dim = deform_fc_dim
        if not no_trans:
            # dcn_v2.py:246-257: a plain MLP (library layers in this standalone module, as DCN.conv_offset_mask)
            self.offset_mask_fc = nn.Sequential(
                nn.Linear(self.pooled_size * self.pooled_size * self.output_dim, self.deform_fc_dim),
                nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, self.deform_fc_dim),
                nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, self.pooled_size * self.pooled_size * 3)
            )
            self.offset_mask_fc[4].weight.data.zero_()
            self.offset_mask_fc[4].bias.data.zero_()

    def forward(self, input, rois):
        offset = input.new()
        if not self.no_trans:
            # dcn_v2.py:262-293: plain pooling, then offsets and masks from the MLP, then deformable pooling * mask
            n = rois.shape[0]
            roi = dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim, True,
                                 self.group_size, self.part_size, self.sample_per_part, self.trans_std)
            offset_mask = self.offset_mask_fc(roi.view(n, -1))
            offset_mask = offset_mask.view(n, 3, self.pooled_size, self.pooled_size)
            o1, o2, mask = torch.chunk(offset_mask, 3, dim=1)
            offset = torch.cat((o1, o2), dim=1)
            mask = torch.sigmoid(mask)
            return dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim,
                                  self.no_trans, self.group_size, self.part_size, self.sample_per_part,
                                  self.trans_std) * mask
        return dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim, self.no_trans,
                              self.group_size, self.part_size, self.sample_per_part, self.trans_std)
