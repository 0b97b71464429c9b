"""CPU oracle for the YOLACT inference path -- TEST INFRASTRUCTURE, never imported by the product.

A restatement of the reference's algorithm, each function citing the reference file:line it follows.
  * conv stack (floating point): torch-CPU fp32 functional ops (F.conv2d, F.batch_norm, ...) driven
    by a reference-format state_dict -- the "plain PyTorch fp32 reference of the same op".
  * priors / decode / Detect (Fast NMS, cross-class) / crop / postprocess / DCNv2 sampling: numpy,
    written from the reference's formulas (index / integer / compare work is bit-exact by construction).

Pinned against the real reference by tests/golden/*.npz (oracle/gen_golden.py, tests/test_oracle_vs_golden.py).
DCNv2: the reference's CUDA extension cannot be built here (THC headers; SURVEY.md section 8c); its
arithmetic is restated from external/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:25-54,125-195 and
dcn_v2_cuda.cu:123-163, cross-checked against torchvision.ops.deform_conv2d (0.26.0) in gen_golden.py
and against the reference's own test.py:32-67 zero-offset identity.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ---------------------------------------------------------------------------------------------
# priors (PredictionModule.make_priors, yolact.py:214-263)
# ---------------------------------------------------------------------------------------------
def make_priors(level_hw, scales, ars, max_size, use_square_anchors):
    data = []
    for (ch, cw), sc in zip(level_hw, scales):
        for j in range(ch):
            for i in range(cw):
                x = (i + 0.5) / cw
                y = (j + 0.5) / ch
                for scale in sc:
                    for ar in ars:
                        a = math.sqrt(ar)          # preapply_sqrt == False (yolact.py:232-233)
                        w = scale * a / max_size   # use_pixel_scales (yolact.py:235-237)
                        h = scale / a / max_size
                        if use_square_anchors:     # yolact.py:243-244
                            h = w
                        data += [x, y, w, h]
    return np.asarray(data, dtype=np.float64).astype(np.float32).reshape(-1, 4)


# ---------------------------------------------------------------------------------------------
# DCNv2 (numpy, vectorised over pixels and channels)
# ---------------------------------------------------------------------------------------------
def dcn_v2_positions(offset, H, W, stride, pad, dil):
    """Sampling positions of every (pixel, tap): h_im, w_im [B,9,Ho,Wo] fp32 and the reference's inside test.  The sum
    is an fp32 sum like the reference's (`const float h_im = h_in + i * dilation_h + offset_h`), and the inside test
    is taken on that rounded value: both decide which corners exist, so they are never widened."""
    offset = np.asarray(offset, np.float32)
    Ho, Wo = offset.shape[2:]
    ho = np.arange(Ho, dtype=np.float32)[:, None]
    wo = np.arange(Wo, dtype=np.float32)[None, :]
    h_im = np.empty((offset.shape[0], 9, Ho, Wo), np.float32)
    w_im = np.empty_like(h_im)
    for k in range(9):
        i, j = divmod(k, 3)
        h_im[:, k] = (ho * stride - pad + i * dil + offset[:, 2 * k]).astype(np.float32)      # im2col_cuda.cu:177
        w_im[:, k] = (wo * stride - pad + j * dil + offset[:, 2 * k + 1]).astype(np.float32)  # :178
    with np.errstate(invalid="ignore"):
        valid = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)                            # :180 (false for NaN)
    return h_im, w_im, valid


def dcn_v2_columns(x, offset, mask, stride, pad, dil, acc=np.float32, with_abs=False):
    """The modulated deformable im2col: x [B,C,H,W], offset [B,18,Ho,Wo] (dh,dw interleaved per tap), mask [B,9,Ho,Wo]
    (already sigmoided) -> columns [B,C,9,Ho,Wo] of dtype `acc`.  Positions, floors and the four fractional weights
    lh, lw, 1-lh, 1-lw are fp32 as in the reference; `acc` is the type of the weight products, the four-corner blend
    and the mask product (np.float32: the reference's arithmetic, np.float64: a high-precision blend of the same
    corners).  with_abs=True also returns sum over the corners of |weight * mask * x|, the scale a rounding error of the
    blend is proportional to."""
    x = np.asarray(x, np.float32)
    mask = np.asarray(mask, np.float32)
    B, C, H, W = x.shape
    h_im, w_im, valid = dcn_v2_positions(offset, H, W, stride, pad, dil)
    Ho, Wo = h_im.shape[2:]
    cols = np.zeros((B, C, 9, Ho, Wo), acc)
    mag = np.zeros((B, C, 9, Ho, Wo), acc) if with_abs else None
    zero = acc(0)
    for b in range(B):
        for k in range(9):
            ok = valid[b, k]
            h = np.where(ok, h_im[b, k], np.float32(0))   # an outside position takes no part below (it may be NaN)
            w = np.where(ok, w_im[b, k], np.float32(0))
            hl = np.floor(h).astype(np.int64)
            wl = np.floor(w).astype(np.int64)
            hh, wh = hl + 1, wl + 1
            lh = (h - hl).astype(np.float32)
            lw = (w - wl).astype(np.float32)
            uh, uw = (1 - lh).astype(np.float32), (1 - lw).astype(np.float32)
            lh, lw, uh, uw = (a.astype(acc) for a in (lh, lw, uh, uw))

            def corner(hi, wi, exists):
                v = x[b][:, np.clip(hi, 0, H - 1), np.clip(wi, 0, W - 1)].astype(acc)  # [C,Ho,Wo]
                return np.where((exists & ok)[None], v, zero)

            v1 = corner(hl, wl, (hl >= 0) & (wl >= 0))                  # :38-48
            v2 = corner(hl, wh, (hl >= 0) & (wh <= W - 1))
            v3 = corner(hh, wl, (hh <= H - 1) & (wl >= 0))
            v4 = corner(hh, wh, (hh <= H - 1) & (wh <= W - 1))
            t1, t2, t3, t4 = (uh * uw) * v1, (uh * lw) * v2, (lh * uw) * v3, (lh * lw) * v4
            val = np.where(ok[None], (t1 + t2 + t3 + t4).astype(acc), zero)                   # :50-53
            m = mask[b, k].astype(acc)[None]
            cols[b, :, k] = val * m                                                          # :189
            if with_abs:
                mag[b, :, k] = np.where(ok[None], np.abs(t1) + np.abs(t2) + np.abs(t3) + np.abs(t4), zero) * np.abs(m)
    return (cols, mag) if with_abs else cols


def dcn_v2_contract(cols, weight, bias, acc=np.float32):
    """columns [B,C,9,Ho,Wo] x weight [Co,C,3,3] + bias [Co] -> [B,Co,Ho,Wo] in `acc` (dcn_v2_cuda.cu:123-163)."""
    B, C, _, Ho, Wo = cols.shape
    Co = weight.shape[0]
    wm = np.asarray(weight, np.float32).reshape(Co, C * 9).astype(acc)
    out = np.einsum("ok,bkp->bop", wm, cols.reshape(B, C * 9, Ho * Wo).astype(acc)).astype(acc)  # :149-163
    out = out + np.asarray(bias, np.float32).astype(acc)[None, :, None]                              # :123-137
    return out.reshape(B, Co, Ho, Wo)


def dcn_v2_forward(x, offset, mask, weight, bias, stride, pad, dil, acc=np.float32):
    """x [B,C,H,W], offset [B,18,Ho,Wo] (dh,dw interleaved per tap), mask [B,9,Ho,Wo] (already
    sigmoided), weight [Co,C,3,3], bias [Co] -> [B,Co,Ho,Wo].  By default everything is fp32 like the reference (using
    scalar_t = float): float64 accumulation of fp32 products is avoided on purpose.  acc=np.float64 keeps the fp32
    sampling geometry and carries the blend and the contraction in float64: the yardstick for the kernels' rounding."""
    return dcn_v2_contract(dcn_v2_columns(x, offset, mask, stride, pad, dil, acc), weight, bias, acc)


# ---------------------------------------------------------------------------------------------
# conv stack (torch CPU fp32)
# ---------------------------------------------------------------------------------------------
class ConvStackOracle(object):
    """Functional Yolact.forward (train-mode outputs: raw loc/conf/mask + priors + proto) from a
    reference-format state_dict.  cfg: yolact_b200.config.Config-like (plain attributes)."""

    def __init__(self, cfg, state_dict):
        self.cfg = cfg
        self.sd = {k: (v.float() if v.is_floating_point() else v) for k, v in state_dict.items()}

    def _conv(self, x, key, stride=1, pad=0):
        return F.conv2d(x, self.sd[key + ".weight"], self.sd.get(key + ".bias"), stride=stride, padding=pad)

    def _bn(self, x, key):  # eval-mode BatchNorm2d, eps 1e-5
        return F.batch_norm(x, self.sd[key + ".running_mean"], self.sd[key + ".running_var"],
                            self.sd[key + ".weight"], self.sd[key + ".bias"], False, 0.0, 1e-5)

    def _dcn(self, x, key, stride):
        # DCN.forward, dcn_v2.py:118-128
        out = self._conv(x, key + ".conv_offset_mask", stride, 1)
        o1, o2, m = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        m = torch.sigmoid(m)
        y = dcn_v2_forward(x.numpy(), offset.numpy(), m.numpy(), self.sd[key + ".weight"].numpy(),
                           self.sd[key + ".bias"].numpy(), stride, 1, 1)
        return torch.from_numpy(y)

    def _uses_dcn(self, stage, j):
        c = self.cfg
        blocks, dl = c.backbone_layers[stage], c.dcn_layers[stage]
        if j == 0:
            return dl >= blocks
        return (j + dl) >= blocks and (j % max(1, c.dcn_interval) == 0)  # backbone.py:112-118

    def backbone(self, x):
        c = self.cfg
        outs = []
        if c.backbone == "resnet":
            # ResNetBackbone.forward, backbone.py:126-139
            x = F.relu(self._bn(self._conv(x, "backbone.conv1", 2, 3), "backbone.bn1"))
            x = F.max_pool2d(x, 3, 2, 1)
            for i, blocks in enumerate(c.backbone_layers):
                for j in range(blocks):
                    n = "backbone.layers.%d.%d" % (i, j)
                    s = (1 if i == 0 else 2) if j == 0 else 1
                    # Bottleneck.forward, backbone.py:37-57
                    o = F.relu(self._bn(self._conv(x, n + ".conv1"), n + ".bn1"))
                    if self._uses_dcn(i, j):
                        o = self._dcn(o, n + ".conv2", s)
                    else:
                        o = self._conv(o, n + ".conv2", s, 1)
                    o = F.relu(self._bn(o, n + ".bn2"))
                    o = self._bn(self._conv(o, n + ".conv3"), n + ".bn3")
                    r = x
                    if j == 0:
                        r = self._bn(self._conv(x, n + ".downsample.0", s, 0), n + ".downsample.1")
                    x = F.relu(o + r)
                outs.append(x)
        else:
            # DarkNetBackbone.forward, backbone.py:299-309; darknetconvlayer :222-233; DarkNetBlock :235-247
            def dconv(x, key, stride=1, pad=0):
                return F.leaky_relu(self._bn(self._conv(x, key + ".0", stride, pad), key + ".1"), 0.1)
            x = dconv(x, "backbone._preconv", 1, 1)
            for i, blocks in enumerate(c.backbone_layers):
                ln = "backbone.layers.%d" % i
                x = dconv(x, ln + ".0", 2, 1)
                for j in range(blocks):
                    n = "%s.%d" % (ln, j + 1)
                    x = dconv(dconv(x, n + ".conv1"), n + ".conv2", 1, 1) + x
                outs.append(x)
        return outs

    def fpn(self, convouts):
        # FPN.forward, yolact.py:311-361 (lat/pred layers stored reversed)
        n = len(convouts)
        out = [None] * n
        x = None
        for i in range(n):
            j = n - 1 - i
            lat = self._conv(convouts[j], "fpn.lat_layers.%d" % i)
            if x is not None:
                x = F.interpolate(x, size=lat.shape[2:], mode="bilinear", align_corners=False)
                x = x + lat
            else:
                x = lat
            out[j] = x
        for i in range(n):
            j = n - 1 - i
            out[j] = F.relu(self._conv(out[j], "fpn.pred_layers.%d" % i, 1, 1))
        for i in range(2):
            out.append(self._conv(out[-1], "fpn.downsample_layers.%d" % i, 2, 1))
        return out

    def proto(self, p3):
        # make_net(cfg.mask_proto_net) + prototype activation (utils/functions.py:163-213, yolact.py:588-599)
        x = F.relu(self._conv(p3, "proto_net.0", 1, 1))
        x = F.relu(self._conv(x, "proto_net.2", 1, 1))
        x = F.relu(self._conv(x, "proto_net.4", 1, 1))
        x = F.relu(F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False))
        x = F.relu(self._conv(x, "proto_net.8", 1, 1))
        x = F.relu(self._conv(x, "proto_net.10"))
        return x.permute(0, 2, 3, 1).contiguous()

    def heads(self, levels):
        # PredictionModule.forward (shared weights), yolact.py:133-212
        c = self.cfg
        loc, conf, mask = [], [], []
        hn = "prediction_layers.0"
        for x in levels:
            B = x.shape[0]
            u = F.relu(self._conv(x, hn + ".upfeature.0", 1, 1))
            loc.append(self._conv(u, hn + ".bbox_layer", 1, 1).permute(0, 2, 3, 1).contiguous().view(B, -1, 4))
            conf.append(self._conv(u, hn + ".conf_layer", 1, 1).permute(0, 2, 3, 1).contiguous().view(B, -1, c.num_classes))
            mask.append(torch.tanh(self._conv(u, hn + ".mask_layer", 1, 1).permute(0, 2, 3, 1).contiguous().view(B, -1, c.mask_dim)))
        return torch.cat(loc, 1), torch.cat(conf, 1), torch.cat(mask, 1)

    def forward(self, x, want_features=False):
        c = self.cfg
        with torch.no_grad():
            outs = self.backbone(x.float())
            sel = [outs[i] for i in c.selected_layers]
            levels = self.fpn(sel)
            proto = self.proto(levels[0])
            loc, conf, mask = self.heads(levels)
        level_hw = [(int(l.shape[2]), int(l.shape[3])) for l in levels]
        priors = make_priors(level_hw, c.pred_scales, c.pred_aspect_ratios, c.max_size, c.use_square_anchors)
        r = {"loc": loc, "conf": conf, "mask": mask, "priors": torch.from_numpy(priors), "proto": proto}
        if want_features:
            r["backbone"] = outs
            r["fpn"] = levels
        return r

    def maskiou(self, masks):
        # FastMaskIoUNet.forward, yolact.py:363-375: masks [n,1,ph,pw] -> [n,80]
        x = masks.float()
        for i in (0, 2, 4, 6, 8):
            x = F.relu(self._conv(x, "maskiou_net.maskiou_net.%d" % i, 2, 0))
        x = F.relu(self._conv(x, "maskiou_net.maskiou_net.10"))
        return F.max_pool2d(x, kernel_size=x.shape[2:]).squeeze(-1).squeeze(-1)


# ---------------------------------------------------------------------------------------------
# Detect (numpy)
# ---------------------------------------------------------------------------------------------
def softmax_rows(x):
    x = np.asarray(x, np.float32)
    m = x.max(axis=-1, keepdims=True)
    e = np.exp(x - m).astype(np.float32)
    return (e / e.sum(axis=-1, keepdims=True, dtype=np.float32)).astype(np.float32)


def decode(loc, priors):
    # box_utils.py:303-310
    loc = np.asarray(loc, np.float32)
    priors = np.asarray(priors, np.float32)
    cxcy = priors[:, :2] + loc[:, :2] * np.float32(0.1) * priors[:, 2:]
    wh = priors[:, 2:] * np.exp(loc[:, 2:] * np.float32(0.2)).astype(np.float32)
    boxes = np.concatenate([cxcy, wh], 1).astype(np.float32)
    boxes[:, :2] -= boxes[:, 2:] / np.float32(2)
    boxes[:, 2:] += boxes[:, :2]
    return boxes


def jaccard(a, b):
    # box_utils.py:32-80 on [n,A,4] x [n,B,4]
    max_xy = np.minimum(a[:, :, None, 2:], b[:, None, :, 2:])
    min_xy = np.maximum(a[:, :, None, :2], b[:, None, :, :2])
    wh = np.clip(max_xy - min_xy, 0, None).astype(np.float32)
    inter = (wh[..., 0] * wh[..., 1]).astype(np.float32)
    area_a = ((a[:, :, 2] - a[:, :, 0]) * (a[:, :, 3] - a[:, :, 1])).astype(np.float32)[:, :, None]
    area_b = ((b[:, :, 2] - b[:, :, 0]) * (b[:, :, 3] - b[:, :, 1])).astype(np.float32)[:, None, :]
    union = (area_a + area_b - inter).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (inter / union).astype(np.float32)


def _stable_desc_order(scores):
    # descending by score, ties by lower index (the contract the CUDA path implements)
    return np.lexsort((np.arange(scores.shape[-1]), -scores.astype(np.float64)))


def cython_nms(dets, thresh):
    """utils/cython_nms.pyx:24-74 restated: dets [n,5] float32 (x1,y1,x2,y2,score) in PIXELS, greedy NMS with
    the +1 area convention; returns the kept indices in ascending index order (np.where).
    Ties in score: lower index first (the pyx uses argsort()[::-1], whose tie order is unspecified)."""
    dets = np.asarray(dets, np.float32)
    x1, y1, x2, y2, sc = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3], dets[:, 4]
    one = np.float32(1)
    areas = ((x2 - x1 + one) * (y2 - y1 + one)).astype(np.float32)
    order = _stable_desc_order(sc)
    n = dets.shape[0]
    suppressed = np.zeros(n, bool)
    for _i in range(n):
        i = order[_i]
        if suppressed[i]:
            continue
        rest = order[_i + 1:]
        rest = rest[~suppressed[rest]]
        if rest.size == 0:
            continue
        xx1 = np.maximum(x1[i], x1[rest])
        yy1 = np.maximum(y1[i], y1[rest])
        xx2 = np.minimum(x2[i], x2[rest])
        yy2 = np.minimum(y2[i], y2[rest])
        w = np.maximum(np.float32(0), (xx2 - xx1 + one).astype(np.float32))
        h = np.maximum(np.float32(0), (yy2 - yy1 + one).astype(np.float32))
        inter = (w * h).astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            ovr = (inter / ((areas[i] + areas[rest]).astype(np.float32) - inter).astype(np.float32)).astype(np.float32)
        suppressed[rest[ovr >= np.float32(thresh)]] = True
    return np.where(~suppressed)[0]


def traditional_nms(boxes, masks, scores, iou_threshold, conf_thresh, max_size, max_dets):
    """Detect.traditional_nms (detection.py:182-228).  boxes [n,4] relative, scores [C-1,n]."""
    boxes = (np.asarray(boxes, np.float32) * np.float32(max_size)).astype(np.float32)    # :194
    idx_lst, cls_lst, scr_lst = [], [], []
    for c in range(scores.shape[0]):
        cls_scores = scores[c]
        conf_mask = cls_scores > np.float32(conf_thresh)                                 # :198
        idx = np.arange(cls_scores.shape[0])[conf_mask]
        cs = cls_scores[conf_mask]
        if cs.shape[0] == 0:
            continue
        keep = cython_nms(np.concatenate([boxes[conf_mask], cs[:, None]], 1), iou_threshold)
        idx_lst.append(idx[keep])
        cls_lst.append(np.full(keep.shape[0], c, np.int64))
        scr_lst.append(cs[keep])
    idx = np.concatenate(idx_lst)
    classes = np.concatenate(cls_lst)
    s = np.concatenate(scr_lst)
    o = _stable_desc_order(s)[:max_dets]                                                 # :219-221
    idx, classes, s = idx[o], classes[o], s[o]
    return (boxes[idx] / np.float32(max_size)).astype(np.float32), masks[idx], classes, s   # :228


def detect_one(loc, conf, mask, priors, conf_thresh=0.05, nms_thresh=0.5, top_k=200, max_dets=100,
               cross_class=False, traditional=False, max_size=550, second_threshold=False):
    """One image.  conf [P,C] softmaxed.  Returns dict(box, mask, class, score) or None
    (Detect.detect + fast_nms / cc_fast_nms / traditional_nms, detection.py:81-228)."""
    conf = np.asarray(conf, np.float32)
    boxes = decode(loc, priors)
    cur = conf[:, 1:].T                                   # [C-1, P]   (detection.py:83)
    conf_scores = cur.max(axis=0)
    keep = conf_scores > np.float32(conf_thresh)          # :86
    scores = cur[:, keep]
    boxes = boxes[keep]
    masks = np.asarray(mask, np.float32)[keep]
    if scores.shape[1] == 0:
        return None                                       # :94-95
    if traditional:
        b, m, c, s = traditional_nms(boxes, masks, scores, nms_thresh, conf_thresh, max_size, max_dets)
        return {"box": b, "mask": m, "class": c.astype(np.int64), "score": s}
    if cross_class:
        # cc_fast_nms, detection.py:111-135
        classes = scores.argmax(axis=0)
        s = scores.max(axis=0)
        idx = _stable_desc_order(s)[:top_k]
        b = boxes[idx]
        iou = np.triu(jaccard(b[None], b[None])[0], k=1)
        iou_max = iou.max(axis=0)
        out = idx[iou_max <= np.float32(nms_thresh)]
        return {"box": boxes[out], "mask": masks[out], "class": classes[out].astype(np.int64), "score": s[out]}
    # fast_nms, detection.py:137-180
    C = scores.shape[0]
    order = np.stack([_stable_desc_order(scores[c]) for c in range(C)])[:, :top_k]   # :138-141
    s = np.take_along_axis(scores, order, axis=1)
    nd = order.shape[1]
    b = boxes[order.reshape(-1)].reshape(C, nd, 4)
    m = masks[order.reshape(-1)].reshape(C, nd, -1)
    iou = jaccard(b, b)
    iou = np.triu(iou, k=1)                                # triu_ on the last two dims (:149)
    iou_max = iou.max(axis=1)                              # column max (:150); NaN propagates like torch.max
    keepm = iou_max <= np.float32(nms_thresh)              # :153
    if second_threshold:
        keepm = keepm & (s > np.float32(conf_thresh))      # :160-161
    classes = np.broadcast_to(np.arange(C)[:, None], keepm.shape)[keepm]
    b, m, s = b[keepm], m[keepm], s[keepm]
    o = _stable_desc_order(s)[:max_dets]                   # :172-174
    return {"box": b[o], "mask": m[o], "class": classes[o].astype(np.int64), "score": s[o]}


# ---------------------------------------------------------------------------------------------
# postprocess (numpy)
# ---------------------------------------------------------------------------------------------
def sanitize_coordinates(x1, x2, img_size, padding=0):
    # box_utils.py:327-346, cast=False
    x1 = (np.asarray(x1, np.float32) * np.float32(img_size)).astype(np.float32)
    x2 = (np.asarray(x2, np.float32) * np.float32(img_size)).astype(np.float32)
    lo = np.minimum(x1, x2)
    hi = np.maximum(x1, x2)
    lo = np.clip(lo - np.float32(padding), 0, None).astype(np.float32)
    hi = np.clip(hi + np.float32(padding), None, np.float32(img_size)).astype(np.float32)
    return lo, hi


def crop(masks, boxes, padding=1):
    # box_utils.py:349-373; masks [h,w,n]
    h, w, n = masks.shape
    x1, x2 = sanitize_coordinates(boxes[:, 0], boxes[:, 2], w, padding)
    y1, y2 = sanitize_coordinates(boxes[:, 1], boxes[:, 3], h, padding)
    rows = np.arange(w, dtype=np.float32).reshape(1, -1, 1)
    cols = np.arange(h, dtype=np.float32).reshape(-1, 1, 1)
    m = (rows >= x1.reshape(1, 1, -1)) & (rows < x2.reshape(1, 1, -1)) & \
        (cols >= y1.reshape(1, 1, -1)) & (cols < y2.reshape(1, 1, -1))
    return masks * m.astype(np.float32)


def bilinear_resize(x, out_h, out_w):
    """[n,h,w] -> [n,out_h,out_w], align_corners=False (ATen upsample_bilinear2d; SURVEY.md Appendix D.12)."""
    x = np.asarray(x, np.float32)
    n, h, w = x.shape

    def table(out, inn):
        scale = np.float32(inn) / np.float32(out)
        d = np.arange(out, dtype=np.float32)
        s = np.maximum(scale * (d + np.float32(0.5)) - np.float32(0.5), np.float32(0)).astype(np.float32)
        i0 = np.minimum(s.astype(np.int64), inn - 1)
        i1 = i0 + (i0 < inn - 1)
        l1 = (s - i0.astype(np.float32)).astype(np.float32)
        return i0, i1, (np.float32(1) - l1).astype(np.float32), l1

    h0, h1, lh0, lh1 = table(out_h, h)
    w0, w1, lw0, lw1 = table(out_w, w)
    top = x[:, h0][:, :, w0] * lw0 + x[:, h0][:, :, w1] * lw1
    bot = x[:, h1][:, :, w0] * lw0 + x[:, h1][:, :, w1] * lw1
    return (top * lh0[None, :, None] + bot * lh1[None, :, None]).astype(np.float32)


def proto_masks(proto, coef, boxes, crop_masks=True):
    # output_utils.py:69-77
    proto = np.asarray(proto, np.float32)
    m = proto @ np.asarray(coef, np.float32).T
    m = (1.0 / (1.0 + np.exp(-m))).astype(np.float32)
    if crop_masks:
        m = crop(m, np.asarray(boxes, np.float32))
    return np.ascontiguousarray(m.transpose(2, 0, 1))


def postprocess_one(det, w, h, crop_masks=True, maskiou_fn=None, rescore_bbox=False):
    """det: dict(box, mask, class, score, proto) numpy.  Returns (classes, scores, boxes, masks) with
    masks float {0,1} [n,h,w], boxes int64 (output_utils.py:58-99)."""
    pm = proto_masks(det["proto"], det["mask"], det["box"], crop_masks)
    scores = det["score"]
    if maskiou_fn is not None:
        miou = maskiou_fn(pm)[np.arange(pm.shape[0]), det["class"]]
        scores = scores * miou if rescore_bbox else [scores, scores * miou]
    masks = (bilinear_resize(pm, h, w) > np.float32(0.5)).astype(np.float32)
    x1, x2 = sanitize_coordinates(det["box"][:, 0], det["box"][:, 2], w)
    y1, y2 = sanitize_coordinates(det["box"][:, 1], det["box"][:, 3], h)
    boxes = np.stack([x1, y1, x2, y2], 1).astype(np.int64)   # .long() truncation
    return det["class"], scores, boxes, masks
