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
