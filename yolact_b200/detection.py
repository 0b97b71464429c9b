"""Detect: drop-in for layers/functions/detection.py:11-228 (fast_nms, cc_fast_nms, traditional_nms) on the CUDA library.

`Detect(num_classes, bkg_label, top_k, conf_thresh, nms_thresh)` and
`detect(predictions, net) -> [{'detection': dict|None, 'net': net}]` keep the reference signature;
`predictions` is the dict Yolact.forward builds: loc [B,P,4], conf [B,P,C] ALREADY SOFTMAXED
(yolact.py:674), mask [B,P,k], priors [P,4], optional proto [B,ph,pw,k].

Tie-breaking contract (the reference's torch.sort is unstable): equal scores are ordered by lower
prior index, then by (class, rank) -- what a stable sort of the reference's tensors would give.
"""
import ctypes

import torch

from . import _lib


class Detect(object):
    def __init__(self, num_classes, bkg_label, top_k, conf_thresh, nms_thresh, cfg=None):
        self.num_classes = num_classes
        self.background_label = bkg_label
        self.top_k = top_k
        self.nms_thresh = nms_thresh
        if nms_thresh <= 0:
            raise ValueError('nms_threshold must be non negative.')  # detection.py:25-26
        self.conf_thresh = conf_thresh
        self.use_cross_class_nms = False
        # The reference's attribute default is False (detection.py:30) but every caller sets it from --fast_nms, whose
        # default is True (eval.py:50,871).  Same default as the reference class: a caller that bypasses eval.py gets
        # traditional_nms, exactly as it would there.
        self.use_fast_nms = False
        self.second_threshold = False   # fast_nms(second_threshold=...) (detection.py:137,160-161); never set by eval.py
        self.max_num_detections = getattr(cfg, "max_num_detections", 100) if cfg is not None else 100
        self.mask_dim = getattr(cfg, "mask_dim", 32) if cfg is not None else 32
        self.max_size = getattr(cfg, "max_size", 550) if cfg is not None else 550   # traditional_nms box scale
        self._handles = {}

    def _handle(self, device):
        if device.type != "cuda":
            raise _lib.YbError("yolact_b200.Detect runs on CUDA (H100) only; there is no CPU path.")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        key = (idx, self.top_k, self.conf_thresh, self.nms_thresh, self.max_num_detections, self.num_classes,
               self.mask_dim, self.max_size)
        if key not in self._handles:
            lib = _lib.load()
            yc = _lib.YbConfig()
            yc.backbone = _lib.YB_BACKBONE_NONE
            yc.num_classes = self.num_classes
            yc.mask_dim = self.mask_dim
            yc.precision = _lib.YB_PREC_F32
            yc.nms_top_k = self.top_k
            yc.nms_conf_thresh = self.conf_thresh
            yc.nms_thresh = self.nms_thresh
            yc.max_num_detections = self.max_num_detections
            yc.max_size = int(self.max_size)
            h = ctypes.c_void_p()
            _lib.check(lib.yb_create(ctypes.byref(yc), idx, ctypes.byref(h)), "yb_create(ops)")
            self._handles[key] = h
        return self._handles[key]

    def nms_mode(self):
        """detection.py:97-106: fast_nms / cc_fast_nms, or traditional_nms when use_fast_nms is False (the
        reference then ignores use_cross_class_nms with a warning)."""
        if not self.use_fast_nms:
            if self.use_cross_class_nms:
                print('Warning: Cross Class Traditional NMS is not implemented.')
            return _lib.YB_NMS_TRADITIONAL
        if self.use_cross_class_nms:
            return _lib.YB_NMS_CROSS_CLASS
        return _lib.YB_NMS_FAST | (_lib.YB_NMS_FLAG_SECOND_THRESHOLD if self.second_threshold else 0)

    def detect_padded(self, loc, conf, mask, priors, conf_is_logits=False):
        """Fixed-size outputs, no host sync: (box [B,M,4], coef [B,M,k], cls [B,M] int64, score [B,M], count [B])."""
        lib = _lib.load()
        dev = loc.device
        self.mask_dim = int(mask.shape[-1])
        h = self._handle(dev)
        B, P = int(loc.shape[0]), int(priors.shape[0])
        loc = loc.contiguous().float()
        conf = conf.contiguous().float().view(B, P, self.num_classes)
        mask = mask.contiguous().float()
        priors = priors.contiguous().float()
        mode = self.nms_mode()
        cc = (mode & 0xFF) == _lib.YB_NMS_CROSS_CLASS
        M = self.top_k if cc else self.max_num_detections
        box = torch.empty(B, M, 4, dtype=torch.float32, device=dev)
        coef = torch.empty(B, M, mask.shape[-1], dtype=torch.float32, device=dev)
        cls = torch.empty(B, M, dtype=torch.int64, device=dev)
        score = torch.empty(B, M, dtype=torch.float32, device=dev)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        _lib.check(lib.yb_detect(h, _lib.ptr(loc), _lib.ptr(conf), _lib.ptr(mask), _lib.ptr(priors), B, P,
                                 1 if conf_is_logits else 0, mode, M, _lib.ptr(box), _lib.ptr(coef),
                                 _lib.ptr(cls), _lib.ptr(score), _lib.ptr(count), _lib.current_stream(dev)),
                   "yb_detect")
        return box, coef, cls, score, count

    def __call__(self, predictions, net):
        loc, conf = predictions['loc'], predictions['conf']
        mask, priors = predictions['mask'], predictions['priors']
        proto = predictions['proto'] if 'proto' in predictions else None
        box, coef, cls, score, count = self.detect_padded(loc, conf, mask, priors)
        out = []
        for b, n in enumerate(count.cpu().tolist()):
            if n == 0:
                out.append({'detection': None, 'net': net})
                continue
            det = {'box': box[b, :n], 'mask': coef[b, :n], 'class': cls[b, :n], 'score': score[b, :n]}
            if proto is not None:
                det['proto'] = proto[b]
            out.append({'detection': det, 'net': net})
        return out

    def __del__(self):
        try:
            lib = _lib.load()
            for h in self._handles.values():
                lib.yb_destroy(h)
        except Exception:
            pass
