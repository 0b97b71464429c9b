"""eval.py's box and mask mAP on the GPU: prep_metrics' matching loop and APDataObject / calc_map (eval.py:386-581,
1006-1032) on the CUDA library.

    ap_data = APData(num_classes=80)                          # one accumulator for every (type, threshold, class) cell
    for each image:
        prep_metrics(ap_data, preds, img, gt, gt_masks, h, w, num_crowd, image_id)   # or ap_data.add(...) on
                                                                                     # postprocess's outputs
    all_maps = calc_map(ap_data)                              # the reference's dict, same values, same table

Per image, the IoU caches come from eval_utils.mask_iou / jaccard (bit-identical to box_utils) and ONE kernel
(yb_eval_match) ranks the detections by score and runs the greedy matching for every class, threshold and type,
appending fixed-size records to a device buffer: no host synchronisation and no `.item()` per IoU.  At the end one
call (yb_eval_ap) sorts the records stably per cell and computes every get_ap in double; get_ap() synchronises once.
The result is the reference's to the bit: same data points in the same push order, same counts, same doubles.
"""
import collections
import ctypes

import numpy as np
import torch

from . import _lib
from .eval_utils import _require_cuda, jaccard, mask_iou, pack_masks
from .output_utils import _ops_handle

IOU_THRESHOLDS = [x / 100 for x in range(50, 100, 5)]   # eval.py:130
TYPES = ("box", "mask")


def _to_device(x, dev):
    """Host array / tensor -> `dev` without a host synchronisation (pinned staging, asynchronous copy)."""
    if isinstance(x, torch.Tensor) and x.is_cuda:
        return x.to(dev)
    t = torch.as_tensor(np.ascontiguousarray(x))
    return t.pin_memory().to(dev, non_blocking=True)


class APData:
    """Device accumulator of ap_data[type][threshold][class] (eval.py:904-907).  Records live in one device buffer in
    push order; `num_gt` per class is a device int64[C] (every cell of a class gains the same count)."""

    def __init__(self, num_classes=80, iou_thresholds=IOU_THRESHOLDS, device=None):
        if not torch.cuda.is_available():
            raise _lib.YbError("yolact_b200.metrics.APData runs on CUDA (H100) only; there is no CPU path.")
        self._init(int(num_classes), [float(t) for t in iou_thresholds], device)

    def _init(self, num_classes, thresholds, device):
        if not 1 <= num_classes <= 2048 or not 1 <= len(thresholds) <= 32:
            raise ValueError("APData: 1 to 2048 classes and 1 to 32 IoU thresholds")
        self.num_classes = num_classes
        self.iou_thresholds = thresholds
        self._device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._thr = (ctypes.c_double * len(thresholds))(*thresholds)
        self._n = 0                                   # records in use
        self._score = torch.empty(0, dtype=torch.float32, device=self._device)
        self._tag = torch.empty(0, dtype=torch.int32, device=self._device)
        self._counts = torch.zeros(num_classes, dtype=torch.int64, device=self._device)
        self._err = torch.zeros(1, dtype=torch.int32, device=self._device)

    @property
    def num_records(self):
        return self._n

    def _reserve(self, extra):
        need = self._n + extra
        if need <= self._score.numel():
            return
        cap = max(need, 2 * self._score.numel(), 4096)
        score = torch.empty(cap, dtype=torch.float32, device=self._device)
        tag = torch.empty(cap, dtype=torch.int32, device=self._device)
        score[:self._n].copy_(self._score[:self._n])
        tag[:self._n].copy_(self._tag[:self._n])
        self._score, self._tag = score, tag

    # ---- one image ----------------------------------------------------------------------------------------------
    def add(self, classes, scores, boxes, masks, gt, gt_masks, h, w, num_crowd):
        """postprocess's outputs for one image at h x w (classes int64 [n], scores [n] or YOLACT++'s [box, mask],
        boxes int64 [n,4] pixels, masks [n,h,w] f32 / u8 or bits [n,h,ceil(w/32)] int32) and the dataset's gt [g,5]
        (relative x1y1x2y2 + class, the last num_crowd rows crowds) and gt_masks [g,h,w] (host or device).
        Asynchronous: nothing waits for the GPU."""
        _require_cuda(classes, "metrics.APData.add")
        n = int(classes.shape[0])
        if n == 0:      # eval.py:405-406: nothing is pushed and the ground truths are not counted
            return
        h, w, num_crowd = int(h), int(w), int(num_crowd)
        dev = self._device
        if classes.device != dev:
            raise ValueError("APData.add: the detections are on %s, the accumulator on %s" % (classes.device, dev))
        gt = np.asarray(gt.cpu() if isinstance(gt, torch.Tensor) else gt)
        gt = gt.reshape(-1, 5) if gt.size else np.zeros((0, 5), np.float32)
        g_all = int(gt.shape[0])
        if not 0 <= num_crowd <= g_all:
            raise ValueError("APData.add: num_crowd %d outside [0, %d]" % (num_crowd, g_all))
        g = g_all - num_crowd
        gt_cls = gt[:, 4].astype(int)
        if g and (gt_cls[:g].min() < 0 or gt_cls[:g].max() >= self.num_classes):
            raise ValueError("APData.add: a ground-truth class is outside [0, %d)" % self.num_classes)
        # box and mask scores
        if isinstance(scores, (list, tuple)):
            box_s, mask_s = scores[0], scores[1]
        else:
            box_s = mask_s = scores
        box_s = box_s.float().contiguous()
        mask_s = mask_s.float().contiguous()
        if box_s.shape[0] != n or mask_s.shape[0] != n or tuple(boxes.shape) != (n, 4):
            raise ValueError("APData.add: classes, scores and boxes disagree on the number of detections")
        # masks: detections and ground truth share one bit-row layout (YB_MASK_BITS: ceil(w/32) words per row)
        wpr = (w + 31) // 32
        if masks.dtype == torch.int32:
            if tuple(masks.shape) != (n, h, wpr):
                raise ValueError("APData.add: bit masks are %s, expected [%d, %d, %d]" % (tuple(masks.shape), n, h, wpr))
            det_bits = masks.reshape(n, h * wpr).contiguous()
        else:
            if tuple(masks.shape[-2:]) != (h, w) or masks.shape[0] != n:
                raise ValueError("APData.add: masks are %s, expected [%d, %d, %d]" % (tuple(masks.shape), n, h, w))
            det_bits = pack_masks(masks.reshape(n, h, w), rows=True).reshape(n, h * wpr)
        gm_shape = tuple(gt_masks.shape)
        if g_all and (len(gm_shape) < 2 or gm_shape[0] != g_all or gm_shape[-2:] != (h, w)):
            raise ValueError("APData.add: gt_masks are %s, expected [%d, %d, %d]" % (gm_shape, g_all, h, w))
        # ground truth to the device: boxes scaled in fp32 (eval.py:390-392), classes, masks
        gt_boxes = gt[:, :4].astype(np.float32)
        gt_boxes[:, [0, 2]] *= np.float32(w)
        gt_boxes[:, [1, 3]] *= np.float32(h)
        gt_boxes = _to_device(gt_boxes, dev) if g_all else torch.zeros(0, 4, device=dev)
        gt_cls_d = _to_device(gt_cls.astype(np.int32), dev) if g_all else torch.zeros(0, dtype=torch.int32, device=dev)
        if g_all:
            gm = _to_device(gt_masks, dev) if not (isinstance(gt_masks, torch.Tensor) and gt_masks.is_cuda) else gt_masks
            gt_bits = pack_masks(gm.reshape(g_all, h, w), rows=True).reshape(g_all, h * wpr)
        else:
            gt_bits = torch.zeros(0, h * wpr, dtype=torch.int32, device=dev)
        boxes_f = boxes.float()

        def bits_iou(b, iscrowd):   # an empty ground-truth side is an empty [n, 0] cache
            if b.shape[0] == 0:
                return torch.empty(n, 0, dtype=torch.float32, device=dev)
            return mask_iou(det_bits, b, iscrowd=iscrowd, packed=True)
        box_iou = jaccard(boxes_f, gt_boxes[:g])
        m_iou = bits_iou(gt_bits[:g], False)
        crowd_box = jaccard(boxes_f, gt_boxes[g:], iscrowd=True)
        crowd_mask = bits_iou(gt_bits[g:], True)
        cls = classes.long().contiguous()
        T = len(self.iou_thresholds)
        self._reserve(2 * T * n)
        lib = _lib.load()
        _lib.check(lib.yb_eval_match(_ops_handle(dev), _lib.ptr(box_iou), _lib.ptr(m_iou), _lib.ptr(crowd_box),
                                     _lib.ptr(crowd_mask), _lib.ptr(cls), _lib.ptr(box_s), _lib.ptr(mask_s), n,
                                     _lib.ptr(gt_cls_d[:g]), g, _lib.ptr(gt_cls_d[g:]), num_crowd, self._thr, T,
                                     self.num_classes, _lib.ptr(self._score[self._n:]), _lib.ptr(self._tag[self._n:]),
                                     _lib.ptr(self._counts), _lib.ptr(self._err), _lib.current_stream(dev)),
                   "yb_eval_match")
        self._n += 2 * T * n

    # ---- results ------------------------------------------------------------------------------------------------
    def get_ap(self):
        """-> (ap float64 [2,T,C], nonempty bool [2,T,C]): APDataObject.get_ap / not is_empty() of every cell, type 0
        box and 1 mask.  One host synchronisation."""
        dev = self._device
        T, C = len(self.iou_thresholds), self.num_classes
        lib = _lib.load()
        nbytes = ctypes.c_int64()
        _lib.check(lib.yb_eval_ap_workspace(self._n, T, C, ctypes.byref(nbytes)), "yb_eval_ap_workspace")
        work = torch.empty(max(1, nbytes.value), dtype=torch.uint8, device=dev)
        ap = torch.empty(2 * T * C, dtype=torch.float64, device=dev)
        nonempty = torch.empty(2 * T * C, dtype=torch.uint8, device=dev)
        _lib.check(lib.yb_eval_ap(_ops_handle(dev), _lib.ptr(self._score), _lib.ptr(self._tag), self._n,
                                  _lib.ptr(self._counts), T, C, _lib.ptr(work), nbytes.value, _lib.ptr(ap),
                                  _lib.ptr(nonempty), _lib.current_stream(dev)), "yb_eval_ap")
        host = torch.cat([ap.view(torch.uint8), nonempty, self._err.view(torch.uint8)]).cpu().numpy()
        err = int(host[-4:].view(np.int32)[0])
        if err & 1:
            raise _lib.YbError("APData: a detection class is outside [0, %d)" % C)
        if err & 2:
            raise _lib.YbError("APData: a ground-truth class is outside [0, %d)" % C)
        ap_h = host[:16 * T * C].view(np.float64).reshape(2, T, C).copy()
        ne_h = host[16 * T * C:18 * T * C].astype(bool).reshape(2, T, C)
        return ap_h, ne_h

    def _host_records(self):
        return self._score[:self._n].cpu().numpy(), self._tag[:self._n].cpu().numpy()

    def data_points(self, type, thr_idx, cls):
        """[(score, is_true)] of one cell in push order (type 'box' / 'mask' or 0 / 1).  Synchronises."""
        y = TYPES.index(type) if isinstance(type, str) else int(type)
        cell = (y * len(self.iou_thresholds) + int(thr_idx)) * self.num_classes + int(cls)
        score, tag = self._host_records()
        sel = (tag >= 0) & ((tag >> 1) == cell)
        return [(float(s), bool(t & 1)) for s, t in zip(score[sel].tolist(), tag[sel].tolist())]

    def num_gt_positives(self):
        """int64 [C]: every cell of class c has num_gt_positives == [c].  Synchronises."""
        return self._counts.cpu().numpy()

    # ---- pickling (eval.py writes ap_data to --ap_data_file and reads it back for --resume) -------------------------
    def __getstate__(self):
        score, tag = self._host_records()
        return {"num_classes": self.num_classes, "iou_thresholds": list(self.iou_thresholds), "score": score,
                "tag": tag, "counts": self._counts.cpu().numpy(), "err": self._err.cpu().numpy()}

    def __setstate__(self, st):
        if not torch.cuda.is_available():
            raise _lib.YbError("yolact_b200.metrics.APData runs on CUDA (H100) only; there is no CPU path.")
        self._init(int(st["num_classes"]), [float(t) for t in st["iou_thresholds"]], None)
        n = int(st["score"].shape[0])
        self._reserve(n)
        if n:
            self._score[:n].copy_(torch.from_numpy(np.ascontiguousarray(st["score"])))
            self._tag[:n].copy_(torch.from_numpy(np.ascontiguousarray(st["tag"])))
        self._n = n
        self._counts.copy_(torch.from_numpy(np.ascontiguousarray(st["counts"])))
        self._err.copy_(torch.from_numpy(np.ascontiguousarray(st["err"])))


def prep_metrics(ap_data, dets, img, gt, gt_masks, h, w, num_crowd, image_id, detections=None, *, crop_masks=True,
                 score_threshold=0.0, postprocess=None):
    """eval.py:386-510 on the matching path: postprocess the image at h x w (bit-packed masks), return early when
    there are no detections, else ap_data.add.  `postprocess` defaults to yolact_b200.postprocess (it must take
    mask_format).  img, image_id and detections are accepted for the reference's call form and unused."""
    if postprocess is None:
        from .output_utils import postprocess
    classes, scores, boxes, masks = postprocess(dets, w, h, crop_masks=crop_masks, score_threshold=score_threshold,
                                                mask_format="bits")
    if classes.size(0) == 0:
        return
    ap_data.add(classes, scores, boxes, masks, gt, gt_masks, h, w, num_crowd)


# ---- prep_metrics for a list of images, straight from the detections --------------------------------------------------
# One image's ground truth as APData.add takes it: boxes fp32 [g_all,4] in pixels (scaled in fp32, eval.py:390-392),
# classes int32 [g_all], masks [g_all,h,w] (host array or device tensor, as given), the crowds the last num_crowd rows.
_GtImage = collections.namedtuple("_GtImage", "boxes cls masks h w g_all num_crowd")


def _gt_image(gt, gt_masks, h, w, num_crowd, num_classes, where):
    """APData.add's checks and staging form of one image's ground truth -> _GtImage; ValueError where APData.add
    raises one."""
    gt = np.asarray(gt.cpu() if isinstance(gt, torch.Tensor) else gt)
    gt = gt.reshape(-1, 5) if gt.size else np.zeros((0, 5), np.float32)
    g_all = int(gt.shape[0])
    if not 0 <= num_crowd <= g_all:
        raise ValueError("%s: num_crowd %d outside [0, %d]" % (where, num_crowd, g_all))
    g = g_all - num_crowd
    gt_cls = gt[:, 4].astype(int)
    if g and (gt_cls[:g].min() < 0 or gt_cls[:g].max() >= num_classes):
        raise ValueError("%s: a ground-truth class is outside [0, %d)" % (where, num_classes))
    gm_shape = tuple(gt_masks.shape) if g_all else ()
    if g_all and (len(gm_shape) < 2 or gm_shape[0] != g_all or gm_shape[-2:] != (h, w)):
        raise ValueError("%s: gt_masks are %s, expected [%d, %d, %d]" % (where, gm_shape, g_all, h, w))
    boxes = gt[:, :4].astype(np.float32)
    boxes[:, [0, 2]] *= np.float32(w)
    boxes[:, [1, 3]] *= np.float32(h)
    return _GtImage(boxes, gt_cls.astype(np.int32), gt_masks if g_all else None, h, w, g_all, num_crowd)


# Where _gt_layout puts each image in the staged ground truth: byte offsets of the three sections of the buffer, and
# per image its first ground-truth row and its first mask word (YB_MASK_BITS words, one [g_all, h, ceil(w/32)] block
# per image in image order).
_GtLayout = collections.namedtuple("_GtLayout", "nbytes box_at cls_at mask_at rows words")


def _gt_layout(images):
    """The staging buffer of a list of _GtImage: boxes fp32 [G,4] | classes int32 [G] | masks uint8 [W,32], G = sum of
    g_all, W = sum of g_all * h * ceil(w/32): each mask row padded with zeros to whole words of 32 pixels, so that
    packing the W rows of 32 bytes gives every image's YB_MASK_BITS block at once.  Sections 16-byte aligned."""
    rows, words = [], []
    G = W = 0
    for im in images:
        rows.append(G)
        words.append(W)
        G += im.g_all
        W += im.g_all * im.h * ((im.w + 31) // 32)
    align = lambda v: (v + 15) // 16 * 16
    box_at = 0
    cls_at = align(16 * G)
    mask_at = align(cls_at + 4 * G)
    return _GtLayout(mask_at + 32 * W, box_at, cls_at, mask_at, rows, words)


def _host_mask_bits(m, g_all, h, w, out):
    """Host masks [g_all,h,w] -> out (bool, same shape, any strides): value > 0.5 after the fp32 conversion pack_masks
    makes, in one pass that writes straight into the staging buffer."""
    m = np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m).reshape(g_all, h, w)
    if m.dtype.kind == "f" and m.dtype != np.float32:
        m = m.astype(np.float32)
    np.greater(m, 0.5, out=out)


def _fill_gt(buf, images, lay):
    """Writes the host parts of images into buf (CPU uint8 tensor [lay.nbytes]) at lay's places; device masks are left
    for the caller (their bytes are zeroed).  -> the indices of the images whose masks are device tensors."""
    G = lay.rows[-1] + images[-1].g_all if images else 0
    host = buf.numpy()
    boxes = host[lay.box_at:lay.box_at + 16 * G].view(np.float32).reshape(G, 4)
    cls = host[lay.cls_at:lay.cls_at + 4 * G].view(np.int32)
    on_device = []
    for j, im in enumerate(images):
        r, wd = lay.rows[j], lay.words[j]
        boxes[r:r + im.g_all] = im.boxes
        cls[r:r + im.g_all] = im.cls
        if not im.g_all:
            continue
        wpr = (im.w + 31) // 32
        dst = host[lay.mask_at + 32 * wd:lay.mask_at + 32 * (wd + im.g_all * im.h * wpr)].reshape(im.g_all, im.h,
                                                                                               32 * wpr)
        dst[:, :, im.w:] = 0
        if isinstance(im.masks, torch.Tensor) and im.masks.is_cuda:
            on_device.append(j)
            dst[:, :, :im.w] = 0
            continue
        _host_mask_bits(im.masks, im.g_all, im.h, im.w, dst[:, :, :im.w].view(np.bool_))
    return on_device


# The caches of one prep_metrics_list call: per image with detections, (image index, n, g, num_crowd, box_iou [n,g],
# mask_iou [n,g], crowd_box_iou [n,nc], crowd_mask_iou [n,nc]); the classes, box and mask scores of those images; their
# ground-truth classes (device int32, per image [g_all]); keep_alive, what the launches read.
_IouList = collections.namedtuple("_IouList", "images cls box_s mask_s gt_cls keep_alive")


def _iou_list(num_classes, dev, preds, sizes, gts, gt_masks, num_crowds, crop_masks, score_threshold,
              where="prep_metrics_list"):
    """Everything prep_metrics_list does before the matching: postprocess without masks, the ground truth in one
    pinned buffer and one H2D copy, one pack launch, one yb_eval_iou_list launch -> _IouList, or None when no image
    has detections."""
    from .output_utils import _postprocess_list
    B = len(preds)
    for name, v in (("sizes", sizes), ("gts", gts), ("gt_masks", gt_masks), ("num_crowds", num_crowds)):
        if len(v) != B:
            raise ValueError("%s: %d %s for %d images" % (where, len(v), name, B))
    from . import config as _config
    live = [d['detection'] for d in preds if d['detection'] is not None]
    if not getattr(_config.cfg, "eval_mask_branch", True) or any('proto' not in d for d in live):
        raise ValueError("%s: the mask mAP needs masks; with cfg.eval_mask_branch off (--detect) the detections carry "
                         "no prototypes" % where)
    for d in live:
        _require_cuda(d['box'], "metrics." + where)
        if d['class'].device != dev:
            raise ValueError("%s: the detections are on %s, the accumulator on %s" % (where, d['class'].device, dev))
    res = _postprocess_list(preds, sizes, crop_masks=crop_masks, score_threshold=score_threshold, mask_format=None)
    sel = [(j, i) for j, i in enumerate(res.live) if int(res.out[i][2].shape[0]) > 0]   # eval.py:405-406
    if not sel:
        return None
    ph, pw, k = res.shape
    images = []
    for _, i in sel:
        h, w = (int(v) for v in sizes[i])
        images.append(_gt_image(gts[i], gt_masks[i], h, w, int(num_crowds[i]), num_classes, where))
    # the ground truth: one pinned buffer, one H2D copy, one pack launch for every image's masks
    lay = _gt_layout(images)
    pinned = torch.empty(max(lay.nbytes, 16), dtype=torch.uint8, pin_memory=True)
    on_device = _fill_gt(pinned, images, lay)
    staged = pinned.to(dev, non_blocking=True)
    for j in on_device:
        im = images[j]
        wpr = (im.w + 31) // 32
        at = lay.mask_at + 32 * lay.words[j]
        dst = staged[at:at + 32 * im.g_all * im.h * wpr].view(im.g_all, im.h, 32 * wpr)
        dst[:, :, :im.w] = im.masks.to(dev).reshape(im.g_all, im.h, im.w).float() > 0.5
    W = lay.words[-1] + images[-1].g_all * images[-1].h * ((images[-1].w + 31) // 32)
    bits = pack_masks(staged[lay.mask_at:lay.mask_at + 32 * W].view(W, 32)) if W else staged[:4].view(torch.int32)
    # the caches: one buffer, per image [box n*g | mask n*g | crowd box n*nc | crowd mask n*nc]
    ns = [int(res.out[i][2].shape[0]) for _, i in sel]
    sizes_c = [2 * n * im.g_all for n, im in zip(ns, images)]
    caches = torch.empty(max(sum(sizes_c), 1), dtype=torch.float32, device=dev)
    items = (_lib.YbEvalIouItem * len(sel))()
    out, cls, box_s, mask_s, gt_cls = [], [], [], [], []
    boxes_base = staged.data_ptr() + lay.box_at
    cls_base = staged.data_ptr() + lay.cls_at
    off = 0
    for j, ((t, i), im, n) in enumerate(zip(sel, images, ns)):
        g, nc = im.g_all - im.num_crowd, im.num_crowd
        views = []
        for m in (g, g, nc, nc):
            views.append(caches[off:off + n * m].view(n, m))
            off += n * m
        pi = res.items[t]
        items[j] = _lib.YbEvalIouItem(pi.proto, pi.coef, pi.box, res.out[i][2].data_ptr(),
                                      bits.data_ptr() + 4 * lay.words[j], boxes_base + 16 * lay.rows[j],
                                      *[v.data_ptr() if v.numel() else None for v in views], n, im.h, im.w, im.g_all,
                                      nc)
        out.append((i, n, g, nc) + tuple(views))
        o = res.out[i]
        cls.append(o[0].long().contiguous())
        box_s.append((o[1][0] if isinstance(o[1], list) else o[1]).float().contiguous())
        mask_s.append((o[1][1] if isinstance(o[1], list) else o[1]).float().contiguous())
        gt_cls.append(cls_base + 4 * lay.rows[j])
    # res.keep_alive holds the inputs res.items points at until this call has read them
    _lib.check(_lib.load().yb_eval_iou_list(_ops_handle(dev, k), items, len(sel), ph, pw, k, 1 if crop_masks else 0,
                                            _lib.current_stream(dev)), "yb_eval_iou_list")
    return _IouList(out, cls, box_s, mask_s, gt_cls, [res.keep_alive, staged, bits, caches, pinned])


def _match_list(ap_data, lst):
    """One yb_eval_match_list call over _iou_list's images: records behind ap_data's, counts into ap_data."""
    dev = ap_data._device
    T = len(ap_data.iou_thresholds)
    total = sum(2 * T * im[1] for im in lst.images)
    ap_data._reserve(total)
    items = (_lib.YbEvalMatchItem * len(lst.images))()
    at = ap_data._n
    ptr = lambda v: v.data_ptr() if v.numel() else None
    for j, (im, cls, bs, ms, gc) in enumerate(zip(lst.images, lst.cls, lst.box_s, lst.mask_s, lst.gt_cls)):
        _, n, g, nc, box_iou, m_iou, crowd_box, crowd_mask = im
        items[j] = _lib.YbEvalMatchItem(ptr(box_iou), ptr(m_iou), ptr(crowd_box), ptr(crowd_mask), cls.data_ptr(),
                                        bs.data_ptr(), ms.data_ptr(), gc if g else None, gc + 4 * g if nc else None,
                                        at, n, g, nc)
        at += 2 * T * n
    _lib.check(_lib.load().yb_eval_match_list(_ops_handle(dev), items, len(lst.images), ap_data._thr, T,
                                              ap_data.num_classes, _lib.ptr(ap_data._score), _lib.ptr(ap_data._tag),
                                              _lib.ptr(ap_data._counts), _lib.ptr(ap_data._err),
                                              _lib.current_stream(dev)), "yb_eval_match_list")
    ap_data._n += total


def prep_metrics_list(ap_data, preds, sizes, gts, gt_masks, num_crowds, *, crop_masks=True, score_threshold=0.0):
    """prep_metrics (eval.py:386-510) for a list of images, straight from the detections: fills ap_data exactly as
    [prep_metrics(ap_data, [p], None, gts[i], gt_masks[i], h_i, w_i, num_crowds[i], i) for i, p in enumerate(preds)]
    would, image i at sizes[i] = (h_i, w_i).  preds: Yolact's output list (one {'net', 'detection'} per image);
    gts [g,5] (relative x1y1x2y2 + class, crowds last), gt_masks [g,h,w] and num_crowds per image, in the dataset's form.

    postprocess_list gives the classes, scores (YOLACT++'s [box, mask] included) and pixel boxes without assembling
    masks; the ground truth of every image goes to the device in one pinned buffer and one H2D copy and is packed in
    one launch; ONE yb_eval_iou_list launch computes every image's four IoU caches from the prototypes, and ONE
    yb_eval_match_list launch runs the matching of every image.  No host sync at score_threshold == 0
    (postprocess_list's one at score_threshold > 0).  ValueError, before anything is added, for lists of different
    lengths, a ground-truth class outside [0, C), num_crowd outside [0, g], gt_masks of the wrong shape, detections
    without masks (cfg.eval_mask_branch off) and detections on another device than ap_data."""
    lst = _iou_list(ap_data.num_classes, ap_data._device, preds, sizes, gts, gt_masks, num_crowds, crop_masks,
                    score_threshold)
    if lst is not None:
        _match_list(ap_data, lst)


def calc_map(ap_data, print_table=True):
    """calc_map (eval.py:1006-1032) from ap_data.get_ap(): {'box': {'all': .., 50: .., ...}, 'mask': {...}}, each
    value round(., 2), and the same table printed."""
    ap, nonempty = ap_data.get_ap()
    thresholds = ap_data.iou_thresholds
    if print_table:
        print("Calculating mAP...")
    all_maps = {}
    for yi, t in enumerate(TYPES):
        row = {"all": 0}
        for ti, thr in enumerate(thresholds):
            vals = ap[yi, ti][nonempty[yi, ti]].tolist()      # class order
            row[int(thr * 100)] = sum(vals) / len(vals) * 100 if vals else 0
        row["all"] = sum(row.values()) / (len(row) - 1)      # 'all' is still 0 in first position
        all_maps[t] = row
    if print_table:
        print_maps(all_maps)
    return {t: {k: round(v, 2) for k, v in row.items()} for t, row in all_maps.items()}


def print_maps(all_maps):
    """The table eval.py prints: one column per key ('all', then .50 ...), one row per type."""
    keys = list(all_maps["box"].keys())
    cell = lambda s: " %5s |" % s
    sep = "-------+" * (len(keys) + 1)
    print()
    print(cell("") + "".join(cell(".%d " % k if isinstance(k, int) else k + " ") for k in keys))
    print(sep)
    for t in TYPES:
        print(cell(t) + "".join(cell("%.2f" % v if v < 100 else "%.1f" % v) for v in all_maps[t].values()))
    print(sep)
    print()


# ---- --output_coco_json (eval.py:300-371, :414-429) -----------------------------------------------------------------
def _category_fn(category_of):
    """category_of: a sequence (or mapping) indexed by class, or a callable (eval.py's get_coco_cat)."""
    return category_of if callable(category_of) else category_of.__getitem__


def append_coco_records(bbox_data, mask_data, category_of, image_id, classes, boxes, box_scores, mask_scores, counts,
                        h, w):
    """prep_metrics' --output_coco_json records of one image (eval.py:420-429, Detections.add_bbox / add_mask), from host
    arrays: classes [n], boxes int64 [n,4] pixels, box / mask scores [n] (fp32 values), counts: n RLE strings (str).
    Rows with (y2-y1)*(x2-x1) > 0 on the int64 boxes append a bbox record to bbox_data and a mask record to mask_data,
    in row order; the records are the reference's dicts, key for key."""
    boxes = np.asarray(boxes, np.int64).reshape(-1, 4)
    with np.errstate(over="ignore"):   # numpy int64 arithmetic wraps, as in eval.py
        keep = (boxes[:, 3] - boxes[:, 1]) * (boxes[:, 2] - boxes[:, 0]) > 0
        bbox = np.concatenate([boxes[:, :2], boxes[:, 2:] - boxes[:, :2]], 1)
    cat = _category_fn(category_of)
    image_id = int(image_id)
    classes = np.asarray(classes).astype(int)
    box_scores = np.asarray(box_scores).astype(float)
    mask_scores = np.asarray(mask_scores).astype(float)
    size = [int(h), int(w)]
    for i in np.flatnonzero(keep).tolist():
        bbox_data.append({"image_id": image_id, "category_id": cat(int(classes[i])),
                          "bbox": [round(float(x) * 10) / 10 for x in bbox[i]], "score": float(box_scores[i])})
        mask_data.append({"image_id": image_id, "category_id": cat(int(classes[i])),
                          "segmentation": {"size": list(size), "counts": counts[i]}, "score": float(mask_scores[i])})


def coco_rle_list(items, num_rows, ph, pw, k, crop_masks=True, extra=(), cap=None, device=None):
    """yb_coco_rle_list over a yb_post_item table (ctypes array) -> (strings, host copies of `extra`, calls).
    strings: one str per row, image by image; extra: device tensors (per-row arrays) copied back in the same D2H copy.
    cap: the initial (runs, characters) arena capacities (an int for both); a too small arena costs exactly one more
    call, with the sizes the first reported.  One host synchronisation, two when an arena was too small."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    B = len(items)
    if cap is None:
        runs_cap = sum(int(it.n) * (2 * int(it.out_w) + 8) for it in items)
        chars_cap = 2 * runs_cap
    elif isinstance(cap, (tuple, list)):
        runs_cap, chars_cap = int(cap[0]), int(cap[1])
    else:
        runs_cap = chars_cap = int(cap)
    extra = [t.contiguous().reshape(-1).view(torch.uint8) for t in extra]
    lib = _lib.load()
    calls = 0
    while True:
        calls += 1
        runs = torch.empty(max(runs_cap, 1), dtype=torch.int32, device=dev)
        chars = torch.empty(max(chars_cap, 1), dtype=torch.uint8, device=dev)
        need = torch.empty(2, dtype=torch.int64, device=dev)
        row_off = torch.empty(max(num_rows, 1), dtype=torch.int64, device=dev)
        row_len = torch.empty(max(num_rows, 1), dtype=torch.int32, device=dev)
        _lib.check(lib.yb_coco_rle_list(_ops_handle(dev, k), items, B, ph, pw, k, 1 if crop_masks else 0,
                                        _lib.ptr(runs), runs_cap, _lib.ptr(chars), chars_cap, _lib.ptr(row_off),
                                        _lib.ptr(row_len), _lib.ptr(need), _lib.current_stream(dev)),
                   "yb_coco_rle_list")
        parts = [need.view(torch.uint8), row_off[:num_rows].view(torch.uint8), row_len[:num_rows].view(torch.uint8)]
        parts += extra + [chars[:chars_cap]]
        host = torch.cat(parts).cpu().numpy()   # the one host synchronisation
        need_h = host[:16].view(np.int64)
        if need_h[0] <= runs_cap and need_h[1] <= chars_cap:
            break
        runs_cap, chars_cap = max(runs_cap, int(need_h[0])), max(chars_cap, int(need_h[1]))
    pos = 16
    off = host[pos:pos + 8 * num_rows].view(np.int64)
    pos += 8 * num_rows
    ln = host[pos:pos + 4 * num_rows].view(np.int32)
    pos += 4 * num_rows
    got = []
    for t in extra:
        got.append(host[pos:pos + t.numel()])
        pos += t.numel()
    text = host[pos:].tobytes()
    strings = [text[o:o + n].decode("ascii") for o, n in zip(off.tolist(), ln.tolist())]
    return strings, got, calls


class Detections:
    """eval.py's Detections (eval.py:300-371) for --output_coco_json: bbox_data / mask_data lists of the reference's
    records, filled from the detections on the GPU.

        dets = Detections(category_of)      # class index -> dataset category id: a sequence or a callable
        dets.add(preds, sizes, image_ids)   # a list of images: Yolact outputs, (h, w) each, their ids
        dets.dump(bbox_det_file, mask_det_file)

    add() takes the pixel boxes, classes and scores (YOLACT++'s [box, mask] scores included) from postprocess_list
    without assembling masks, then ONE yb_coco_rle_list launch writes every row's RLE string, and one D2H copy brings
    the strings and the per-row arrays back."""

    def __init__(self, category_of):
        self.bbox_data = []
        self.mask_data = []
        self.category_of = category_of

    def add(self, preds, sizes, image_ids, crop_masks=True, score_threshold=0, cap=None):
        """prep_metrics' --output_coco_json branch (eval.py:414-429) for every image of preds (postprocess_list's
        det_output: one {'net', 'detection'} per image), image i at sizes[i] = (h, w) with id image_ids[i].  One host
        synchronisation (two when the string arena overflows, plus postprocess_list's one when score_threshold > 0);
        returns the number of yb_coco_rle_list calls."""
        from .output_utils import _postprocess_list
        if len(image_ids) != len(preds):
            raise ValueError("Detections.add: %d image ids for %d images" % (len(image_ids), len(preds)))
        for d in preds:
            if d['detection'] is not None:
                _require_cuda(d['detection']['box'], "metrics.Detections.add")
        from . import config as _config
        if not getattr(_config.cfg, "eval_mask_branch", True) or any(
                d['detection'] is not None and 'proto' not in d['detection'] for d in preds):
            raise ValueError("Detections.add: --output_coco_json needs masks; with cfg.eval_mask_branch off (--detect) "
                             "the detections carry no prototypes to encode")
        res = _postprocess_list(preds, sizes, crop_masks=crop_masks, score_threshold=score_threshold, mask_format=None)
        if not res.live:   # no image has detections (eval.py:410-411)
            return 0
        ph, pw, k = res.shape
        out = [res.out[i] for i in res.live]
        cls = [o[0].long() for o in out]
        box_s = [(o[1][0] if isinstance(o[1], list) else o[1]).float() for o in out]
        mask_s = [(o[1][1] if isinstance(o[1], list) else o[1]).float() for o in out]
        boxes = [o[2] for o in out]
        ns = [int(b.shape[0]) for b in boxes]
        extra = [torch.cat(t) for t in (cls, boxes, box_s, mask_s)]
        # res.keep_alive holds the inputs res.items points at until this call has read them
        strings, (cls_h, box_h, bs_h, ms_h), calls = coco_rle_list(res.items, sum(ns), ph, pw, k, crop_masks, extra,
                                                                   cap, extra[0].device)
        cls_h, box_h = cls_h.view(np.int64), box_h.view(np.int64).reshape(-1, 4)
        bs_h, ms_h = bs_h.view(np.float32), ms_h.view(np.float32)
        r = 0
        for i, n in zip(res.live, ns):
            h, w = (int(v) for v in sizes[i])
            append_coco_records(self.bbox_data, self.mask_data, self.category_of, image_ids[i], cls_h[r:r + n],
                                box_h[r:r + n], bs_h[r:r + n], ms_h[r:r + n], strings[r:r + n], h, w)
            r += n
        return calls

    def dump(self, bbox_det_file, mask_det_file):
        """Detections.dump (eval.py:332-340): json.dump of bbox_data and mask_data, the same bytes."""
        import json
        for data, path in ((self.bbox_data, bbox_det_file), (self.mask_data, mask_det_file)):
            with open(path, "w") as f:
                json.dump(data, f)
