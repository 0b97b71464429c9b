"""Yolact: drop-in for the reference's `Yolact` nn.Module (yolact.py:379-676).

Same surface: `Yolact()` reads the package `cfg`; `.load_weights(path)`, `.state_dict()` with the
reference's key names (SURVEY.md Appendix B), `.eval()/.train()/.cuda()`, `net(x)` with x fp32
[B,3,H,W] NCHW; in eval mode returns `[{'detection': dict|None, 'net': net}] * B`
(layers/functions/detection.py:73-76), in train mode the raw dict `loc/conf/mask/priors/proto`
(yolact.py:639-647).  `.detect` is a `Detect` whose `use_fast_nms` / `use_cross_class_nms` flags
eval.py assigns (eval.py:871-872); `.maskiou_net` exists for YOLACT++ configs.

Everything numerical happens in libyolact_b200.so through the C ABI (include/yolact_b200.h); the
nn.Module tree below only HOLDS parameters under the reference's names -- its layers are never
called.  There is no PyTorch/CPU fallback: without the CUDA library on an H100 forward() raises.
"""
import ctypes

import torch
import torch.nn as nn

from . import _lib
from . import config as _config
from .augmentations import frame_geometry, frame_list_geometry, transform_mode
from .detection import Detect


# ---------------------------------------------------------------------------------------------
# parameter holders (names == reference state_dict keys)
# ---------------------------------------------------------------------------------------------
class _DCNParams(nn.Module):
    """Parameters of dcn_v2.DCN (external/DCNv2/dcn_v2.py:57-111)."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        self.bias = nn.Parameter(torch.zeros(cout))
        self.conv_offset_mask = nn.Conv2d(cin, 27, 3, stride=stride, padding=1, bias=True)
        n = cin * 9
        self.weight.data.uniform_(-1.0 / n ** 0.5, 1.0 / n ** 0.5)
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()


class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride, downsample, use_dcn):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _DCNParams(planes, planes, stride) if use_dcn else \
            nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False),
                                            nn.BatchNorm2d(planes * 4))


def _block_uses_dcn(blocks, dcn_layers, dcn_interval, j):
    # backbone.py:112-118
    if j == 0:
        return dcn_layers >= blocks
    return (j + dcn_layers) >= blocks and (j % dcn_interval == 0)


class _ResNetParams(nn.Module):
    def __init__(self, layers, dcn_layers, dcn_interval):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.layers = nn.ModuleList()
        self.channels = []
        inplanes = 64
        for i, blocks in enumerate(layers):
            planes = 64 << i
            stride = 1 if i == 0 else 2
            mods = []
            for j in range(blocks):
                mods.append(_Bottleneck(inplanes, planes, stride if j == 0 else 1, j == 0,
                                        _block_uses_dcn(blocks, dcn_layers[i], max(1, dcn_interval), j)))
                inplanes = planes * 4
            self.layers.append(nn.Sequential(*mods))
            self.channels.append(planes * 4)


def _dark_conv(cin, cout, k, **kw):
    return nn.Sequential(nn.Conv2d(cin, cout, k, bias=False, **kw), nn.BatchNorm2d(cout), nn.Identity())


class _DarkBlock(nn.Module):
    def __init__(self, cin, ch):
        super().__init__()
        self.conv1 = _dark_conv(cin, ch, 1)
        self.conv2 = _dark_conv(ch, ch * 2, 3, padding=1)


class _DarkNetParams(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self._preconv = _dark_conv(3, 32, 3, padding=1)
        self.layers = nn.ModuleList()
        self.channels = []
        cin = 32
        for i, n in enumerate(layers):
            ch = 32 << i
            mods = [_dark_conv(cin, ch * 2, 3, padding=1, stride=2)]
            cin = ch * 2
            mods += [_DarkBlock(cin, ch) for _ in range(n)]
            self.layers.append(nn.Sequential(*mods))
            self.channels.append(cin)


class _FPNParams(nn.Module):
    def __init__(self, in_channels, feats):
        super().__init__()
        self.lat_layers = nn.ModuleList([nn.Conv2d(c, feats, 1) for c in reversed(in_channels)])
        self.pred_layers = nn.ModuleList([nn.Conv2d(feats, feats, 3, padding=1) for _ in in_channels])
        self.downsample_layers = nn.ModuleList([nn.Conv2d(feats, feats, 3, padding=1, stride=2) for _ in range(2)])


class _HeadParams(nn.Module):
    def __init__(self, feats, num_priors, num_classes, mask_dim):
        super().__init__()
        self.upfeature = nn.Sequential(nn.Conv2d(feats, feats, 3, padding=1), nn.Identity())
        self.bbox_layer = nn.Conv2d(feats, num_priors * 4, 3, padding=1)
        self.conf_layer = nn.Conv2d(feats, num_priors * num_classes, 3, padding=1)
        self.mask_layer = nn.Conv2d(feats, num_priors * mask_dim, 3, padding=1)


class FastMaskIoUNet(nn.Module):
    """YOLACT++ mask re-scoring head (yolact.py:363-375); forward runs on the CUDA library."""

    def __init__(self, owner, num_classes):
        super().__init__()
        chans = [1, 8, 16, 32, 64, 128]
        mods = []
        for i in range(5):
            mods += [nn.Conv2d(chans[i], chans[i + 1], 3, stride=2), nn.Identity()]
        mods += [nn.Conv2d(128, num_classes - 1, 1), nn.Identity()]
        self.maskiou_net = nn.Sequential(*mods)
        self._owner = [owner]  # not registered as a submodule

    def forward(self, x):
        net = self._owner[0]
        n, _, ph, pw = x.shape
        out = torch.empty(n, net.cfg.num_classes - 1, device=x.device, dtype=torch.float32)
        if n > 0:
            lib = _lib.load()
            x = x.contiguous().float()
            _lib.check(lib.yb_maskiou(net._handle_for(x.device), _lib.ptr(x), n, ph, pw, None, _lib.ptr(out),
                                      _lib.current_stream(x.device)), "yb_maskiou")
        return out


# ---------------------------------------------------------------------------------------------
def make_yb_config(c, precision):
    yc = _lib.YbConfig()
    yc.backbone = _lib.YB_BACKBONE_RESNET if c.backbone == "resnet" else _lib.YB_BACKBONE_DARKNET
    yc.num_stages = len(c.backbone_layers)
    for i, v in enumerate(c.backbone_layers):
        yc.layers[i] = v
    for i, v in enumerate(c.dcn_layers):
        yc.dcn_layers[i] = v
    yc.dcn_interval = c.dcn_interval
    for i, v in enumerate(c.selected_layers):
        yc.selected_layers[i] = v
    yc.max_size = c.max_size
    yc.num_classes = c.num_classes
    yc.mask_dim = c.mask_dim
    yc.fpn_features = c.fpn_features
    yc.num_scales = len(c.pred_scales[0])
    for l in range(5):
        for s, v in enumerate(c.pred_scales[l]):
            yc.scales[l][s] = float(v)
            yc.scales_f64[l][s] = float(v)     # un-rounded: the reference computes the anchors in doubles
    yc.num_ars = len(c.pred_aspect_ratios)
    for i, v in enumerate(c.pred_aspect_ratios):
        yc.ars[i] = float(v)
        yc.ars_f64[i] = float(v)
    yc.use_square_anchors = 1 if c.use_square_anchors else 0
    yc.use_maskiou = 1 if c.use_maskiou else 0
    yc.precision = precision
    yc.nms_top_k = c.nms_top_k
    yc.nms_conf_thresh = c.nms_conf_thresh
    yc.nms_thresh = c.nms_thresh
    yc.max_num_detections = c.max_num_detections
    return yc


class Yolact(nn.Module):
    """See the module docstring.  `precision` (yb_precision in include/yolact_b200.h):
      'f16x3' (default) split-precision tensor-core -- fp16 hi+lo operand pairs, three MMA passes, fp32-equivalent results
              (boxes / scores / masks within 1e-3 of the fp32 reference, identical class ids);
      'f16tc' single-pass fp16 tensor-core -- faster conv stack, head tensors within ~2e-3 of range;
      'f32'   fp32 on CUDA cores (slow second opinion)."""

    def __init__(self, cfg=None, precision="f16x3"):
        super().__init__()
        c = (cfg or _config.cfg).copy()
        self.cfg = c
        # side effects the reference's constructor has on its global cfg (yolact.py:425,445)
        _config.cfg.mask_dim = c.mask_dim
        _config.cfg.num_heads = 5
        self.precision = _lib.PRECISIONS[precision]
        self.precision_name = precision

        if c.backbone == "resnet":
            self.backbone = _ResNetParams(c.backbone_layers, c.dcn_layers, c.dcn_interval)
        else:
            self.backbone = _DarkNetParams(c.backbone_layers)
        src = [self.backbone.channels[i] for i in c.selected_layers]
        f = c.fpn_features
        # proto_net indices follow make_net's [layer, ReLU] pairs (utils/functions.py:163-213, config.py:691)
        self.proto_net = nn.Sequential(
            nn.Conv2d(f, 256, 3, padding=1), nn.Identity(), nn.Conv2d(256, 256, 3, padding=1), nn.Identity(),
            nn.Conv2d(256, 256, 3, padding=1), nn.Identity(), nn.Identity(), nn.Identity(),
            nn.Conv2d(256, 256, 3, padding=1), nn.Identity(), nn.Conv2d(256, c.mask_dim, 1))
        if c.use_maskiou:
            self.maskiou_net = FastMaskIoUNet(self, c.num_classes)
        self.fpn = _FPNParams(src, f)
        self.num_priors = len(c.pred_aspect_ratios) * len(c.pred_scales[0])
        self.prediction_layers = nn.ModuleList(
            [_HeadParams(f, self.num_priors, c.num_classes, c.mask_dim)] + [nn.Module() for _ in range(4)])
        self.semantic_seg_conv = nn.Conv2d(f, c.num_classes - 1, 1)  # training-only, kept for key parity
        self.detect = Detect(c.num_classes, bkg_label=0, top_k=c.nms_top_k, conf_thresh=c.nms_conf_thresh,
                             nms_thresh=c.nms_thresh, cfg=c)
        self._handles = {}      # device index -> yb_handle
        self._version = 1       # bumped whenever the parameters may have changed
        self._pushed = {}       # device index -> version of the weights that handle holds
        self._detect_pushed = {}  # device index -> (top_k, conf_thresh, nms_thresh, max_num_detections) the handle uses

    # ---- weights ---------------------------------------------------------------------------------
    def save_weights(self, path):
        torch.save(self.state_dict(), path)

    def load_weights(self, path):
        """Same filtering as the reference (yolact.py:477-490)."""
        state_dict = torch.load(path, map_location="cpu")
        for key in list(state_dict.keys()):
            if key.startswith("backbone.layer") and not key.startswith("backbone.layers"):
                del state_dict[key]
            if key.startswith("fpn.downsample_layers."):
                if int(key.split(".")[2]) >= 2:
                    del state_dict[key]
        self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict, strict=True):
        r = super().load_state_dict(state_dict, strict=strict)
        self._version += 1
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._version += 1
        return r

    def mark_weights_dirty(self):
        """Call after modifying parameters in place; the next forward on each device re-uploads them."""
        self._version += 1

    def train(self, mode=True):
        super().train(mode)
        return self

    def _handle_for(self, device):
        if device.type != "cuda":
            raise _lib.YbError("yolact_b200 runs on CUDA (H100) only; got a tensor on %s. There is no CPU path." % device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        lib = _lib.load()
        if idx not in self._handles:
            h = ctypes.c_void_p()
            yc = make_yb_config(self.cfg, self.precision)
            _lib.check(lib.yb_create(ctypes.byref(yc), idx, ctypes.byref(h)), "yb_create")
            self._handles[idx] = h
        h = self._handles[idx]
        if self._pushed.get(idx) != self._version:     # per device: every handle re-syncs on its next call
            self._push_weights(h)
            self._pushed[idx] = self._version
        return h

    def _push_weights(self, h):
        lib = _lib.load()
        for name, t in self.state_dict().items():
            if name.endswith("num_batches_tracked") or name.startswith("semantic_seg_conv"):
                continue
            t = t.detach().to("cpu", torch.float32).contiguous()
            shape = (ctypes.c_int64 * max(1, t.dim()))(*t.shape)
            _lib.check(lib.yb_load_weight(h, name.encode(), ctypes.c_void_p(t.data_ptr()), shape, t.dim()),
                       "yb_load_weight(%s)" % name)
        _lib.check(lib.yb_finalize_weights(h), "yb_finalize_weights")

    def __del__(self):
        try:
            lib = _lib.load()
            for h in self._handles.values():
                lib.yb_destroy(h)
        except Exception:
            pass

    # ---- introspection ---------------------------------------------------------------------------
    def launch_count(self):
        lib = _lib.load()
        return sum(int(lib.yb_launch_count(h)) for h in self._handles.values())

    def profile_conv_stack(self, x):
        """Per-op device times (ms) of one eager conv-stack pass: [(layer name, ms)], CUDA events."""
        x = self._check_input(x)
        lib = _lib.load()
        h = self._handle_for(x.device)
        B, _, H, W = x.shape
        st = _lib.current_stream(x.device)
        _lib.check(lib.yb_forward(h, _lib.ptr(x), B, H, W, None, None, None, None, st), "yb_forward")
        _lib.check(lib.yb_set_profiling(h, 1), "yb_set_profiling")
        try:
            _lib.check(lib.yb_forward(h, _lib.ptr(x), B, H, W, None, None, None, None, st), "yb_forward")
        finally:
            lib.yb_set_profiling(h, 0)
        buf = ctypes.create_string_buffer(1 << 20)
        _lib.check(lib.yb_last_forward_profile(h, buf, len(buf)), "yb_last_forward_profile")
        out = []
        for line in buf.value.decode().splitlines():
            name, ms = line.rsplit(",", 1)
            out.append((name, float(ms)))
        return out

    def num_priors_for(self, h, w, device=None):
        lib = _lib.load()
        n = ctypes.c_int64()
        dev = device or torch.device("cuda", torch.cuda.current_device())
        _lib.check(lib.yb_num_priors(self._handle_for(dev), h, w, ctypes.byref(n), None), "yb_num_priors")
        return n.value

    def debug_feature(self, which, device):
        lib = _lib.load()
        h = self._handle_for(device)
        chw = (ctypes.c_int32 * 3)()
        _lib.check(lib.yb_debug_feature(h, which, None, chw, _lib.current_stream(device)), "yb_debug_feature")
        B = self._last_B
        out = torch.empty(B, chw[0], chw[1], chw[2], device=device, dtype=torch.float32)
        _lib.check(lib.yb_debug_feature(h, which, _lib.ptr(out), chw, _lib.current_stream(device)), "yb_debug_feature")
        return out

    # ---- forward ---------------------------------------------------------------------------------
    def forward_raw(self, x):
        """Conv stack only -> dict(loc, conf [raw logits], mask, priors, proto) (yolact.py:639-647)."""
        x = self._check_input(x)
        lib = _lib.load()
        h = self._handle_for(x.device)
        B, _, H, W = x.shape
        P = self.num_priors_for(H, W, x.device)
        ph, pw = ctypes.c_int32(), ctypes.c_int32()
        _lib.check(lib.yb_proto_size(h, H, W, ctypes.byref(ph), ctypes.byref(pw)), "yb_proto_size")
        c = self.cfg
        o = dict(device=x.device, dtype=torch.float32)
        loc = torch.empty(B, P, 4, **o)
        conf = torch.empty(B, P, c.num_classes, **o)
        mask = torch.empty(B, P, c.mask_dim, **o)
        proto = torch.empty(B, ph.value, pw.value, c.mask_dim, **o)
        priors = torch.empty(P, 4, **o)
        st = _lib.current_stream(x.device)
        _lib.check(lib.yb_forward(h, _lib.ptr(x), B, H, W, _lib.ptr(loc), _lib.ptr(conf), _lib.ptr(mask),
                                  _lib.ptr(proto), st), "yb_forward")
        _lib.check(lib.yb_priors(h, H, W, _lib.ptr(priors), st), "yb_priors")
        self._last_B = B
        return {"loc": loc, "conf": conf, "mask": mask, "priors": priors, "proto": proto}

    def forward_conv_only(self, x):
        """Conv stack (one CUDA graph) with no copy-out: what bench.py times for the conv roofline."""
        x = self._check_input(x)
        lib = _lib.load()
        B, _, H, W = x.shape
        _lib.check(lib.yb_forward(self._handle_for(x.device), _lib.ptr(x), B, H, W, None, None, None, None,
                                  _lib.current_stream(x.device)), "yb_forward")

    def infer_padded(self, x, cross_class=None):
        """Fused forward + Detect with fixed-size outputs and NO host sync:
        (box [B,M,4], coef [B,M,k], cls int64 [B,M], score [B,M], count int32 [B], proto [B,ph,pw,k])."""
        x = self._check_input(x)
        lib = _lib.load()
        h = self._handle_for(x.device)
        B, _, H, W = x.shape
        mode, M, out = self._detect_outputs(h, x.device, B, H, W, cross_class)
        box, coef, cls, score, count, proto = out
        _lib.check(lib.yb_infer(h, _lib.ptr(x), B, H, W, mode, M, _lib.ptr(box), _lib.ptr(coef),
                                _lib.ptr(cls), _lib.ptr(score), _lib.ptr(count), _lib.ptr(proto),
                                _lib.current_stream(x.device)), "yb_infer")
        self._last_B = B
        return out

    def infer_frames(self, frames, cross_class=None):
        """infer_padded(FastBaseTransform(self.cfg)(frames)) as one call, bit for bit, with no host sync and one CUDA
        graph per network input size whatever the frame size; the frames are read in place.
        frames: CUDA uint8 [B,h,w,3] BGR, any size; the network input size and the transform come from self.cfg
        (max_size, preserve_aspect_ratio, normalize / subtract_means / to_float) as in FastBaseTransform.  In the
        tensor-core precisions the resize and transform run inside the stem kernel: no fp32 input tensor is written.
        frames may also be a list or tuple of B CUDA uint8 [h_i,w_i,3] BGR frames of different sizes (a folder of
        images): the same as infer_padded(torch.cat([FastBaseTransform(self.cfg)(f[None]) for f in frames])), from one
        call and one CUDA graph whatever the sizes; the frames are read in place."""
        return self._infer_frames(frames, cross_class)[0]

    def forward_frames(self, frames):
        """forward(FastBaseTransform(self.cfg)(frames)) in eval mode, from uint8 frames (see infer_frames; a list of
        differently sized frames too): [{'detection': dict|None, 'net': net}] * B, which postprocess takes unchanged
        (postprocess(preds, w_i, h_i, i) for image i of a list)."""
        if self.training:
            raise RuntimeError("Yolact.forward_frames is the eval-mode path; call net.eval() first")
        out, oh, ow = self._infer_frames(frames, None)
        _config.cfg._tmp_img_h, _config.cfg._tmp_img_w = oh, ow   # the network input size, as forward sets it
        return self._detection_list(out)

    def _infer_frames(self, frames, cross_class):
        if isinstance(frames, (list, tuple)):
            return self._infer_frame_list(frames, cross_class)
        B, H, W, oh, ow = frame_geometry(self.cfg, frames, "Yolact.infer_frames")
        if frames.dtype != torch.uint8:
            raise ValueError("Yolact.infer_frames takes uint8 frames; run float frames through "
                             "FastBaseTransform and infer_padded")
        x = frames.contiguous()
        lib = _lib.load()
        h = self._handle_for(x.device)
        mode, M, out = self._detect_outputs(h, x.device, B, oh, ow, cross_class)
        box, coef, cls, score, count, proto = out
        mean = (ctypes.c_float * 3)(*_config.MEANS)
        std = (ctypes.c_float * 3)(*_config.STD)
        _lib.check(lib.yb_infer_frames(h, _lib.ptr(x), B, H, W, oh, ow, transform_mode(self.cfg), mean, std, mode, M,
                                       _lib.ptr(box), _lib.ptr(coef), _lib.ptr(cls), _lib.ptr(score), _lib.ptr(count),
                                       _lib.ptr(proto), _lib.current_stream(x.device)), "yb_infer_frames")
        self._last_B = B
        return out, oh, ow

    def _infer_frame_list(self, frames, cross_class):
        hw, oh, ow = frame_list_geometry(self.cfg, frames, "Yolact.infer_frames")
        if any(f.dtype != torch.uint8 for f in frames):
            raise ValueError("Yolact.infer_frames takes uint8 frames; run float frames through "
                             "FastBaseTransform and infer_padded")
        xs = [f.contiguous() for f in frames]   # held until the call has enqueued its reads of them
        B = len(xs)
        device = xs[0].device
        lib = _lib.load()
        h = self._handle_for(device)
        mode, M, out = self._detect_outputs(h, device, B, oh, ow, cross_class)
        mean = (ctypes.c_float * 3)(*_config.MEANS)
        std = (ctypes.c_float * 3)(*_config.STD)
        ptrs = (ctypes.c_void_p * B)(*[x.data_ptr() for x in xs])
        sizes = (ctypes.c_int32 * (2 * B))(*[v for s in hw for v in s])
        _lib.check(lib.yb_infer_frame_list(h, ptrs, sizes, B, oh, ow, transform_mode(self.cfg), mean, std, mode, M,
                                           *[_lib.ptr(t) for t in out], _lib.current_stream(device)),
                   "yb_infer_frame_list")
        self._last_B = B
        return out, oh, ow

    def _detect_outputs(self, h, device, B, H, W, cross_class):
        """The NMS mode, the padded row count M and the empty output tensors of one yb_infer call on [B,3,H,W]."""
        lib = _lib.load()
        c = self.cfg
        if cross_class is None:
            mode = self.detect.nms_mode()   # fast_nms | cc_fast_nms | traditional_nms (--fast_nms=False)
        else:
            mode = _lib.YB_NMS_CROSS_CLASS if cross_class else _lib.YB_NMS_FAST
        # net.detect's attributes are live in the reference (detection.py:17-31): push them when they changed
        d = self.detect
        dkey = (int(d.top_k), float(d.conf_thresh), float(d.nms_thresh), int(d.max_num_detections))
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._detect_pushed.get(idx) != dkey:
            _lib.check(lib.yb_set_detect_params(h, *dkey), "yb_set_detect_params")
            self._detect_pushed[idx] = dkey
        M = dkey[0] if (mode & 0xFF) == _lib.YB_NMS_CROSS_CLASS else dkey[3]
        ph, pw = ctypes.c_int32(), ctypes.c_int32()
        _lib.check(lib.yb_proto_size(h, H, W, ctypes.byref(ph), ctypes.byref(pw)), "yb_proto_size")
        o = dict(device=device)
        box = torch.empty(B, M, 4, dtype=torch.float32, **o)
        coef = torch.empty(B, M, c.mask_dim, dtype=torch.float32, **o)
        cls = torch.empty(B, M, dtype=torch.int64, **o)
        score = torch.empty(B, M, dtype=torch.float32, **o)
        count = torch.empty(B, dtype=torch.int32, **o)
        proto = torch.empty(B, ph.value, pw.value, c.mask_dim, dtype=torch.float32, **o) if c.eval_mask_branch else None
        return mode, M, (box, coef, cls, score, count, proto)

    def forward(self, x):
        _config.cfg._tmp_img_h, _config.cfg._tmp_img_w = int(x.shape[2]), int(x.shape[3])  # yolact.py:567-568
        if self.training:
            return self.forward_raw(x)
        return self._detection_list(self.infer_padded(x))

    def _detection_list(self, padded):
        """infer_padded's outputs -> the eval-mode list of {'detection', 'net'} (detection.py:73-95)."""
        box, coef, cls, score, count, proto = padded
        # the fixed-size tensors the per-image views below are cut from: what a multi-GPU caller hands to
        # parallel.gather_detections (one pack kernel + one all_gather) instead of re-padding the views
        self.last_padded_detections = (box, coef, cls, score, count)
        counts = count.cpu().tolist()  # the only host sync: Detect's output is variable-size by contract
        out = []
        for b, n in enumerate(counts):
            if n == 0:
                out.append({"detection": None, "net": self})  # detection.py:94-95
                continue
            det = {"box": box[b, :n], "mask": coef[b, :n], "class": cls[b, :n], "score": score[b, :n]}
            if proto is not None:
                det["proto"] = proto[b]
            out.append({"detection": det, "net": self})
        return out

    @staticmethod
    def _check_input(x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("Yolact.forward expects [B,3,H,W], got %s" % (tuple(x.shape),))
        if not x.is_cuda:
            raise _lib.YbError("yolact_b200 runs on CUDA (H100) only; input is on %s. There is no CPU path." % x.device)
        return x.contiguous().float()
