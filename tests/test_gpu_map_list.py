"""prep_metrics_list: eval.py's mAP bookkeeping for a list of images straight from the detections (yb_eval_iou_list +
yb_eval_match_list) against the per-image path (postprocess(mask_format='bits') + mask_iou / jaccard + yb_eval_match):
the four IoU caches bit for bit, the records, counts and get_ap exactly; the matching alone on the real reference's
golden; poisoned outputs between guard bands; the refusals; one launch of each kernel per list."""
import ctypes

import numpy as np
import pytest
import torch

import yolact_b200
from tests import test_gpu_mask_edges as ME
from tests.map_oracle import golden_all_maps, golden_images, golden_points
from tests.test_gpu_frames import make_net
from tests.test_gpu_map import _assert_equal_to, _golden
from tests.test_gpu_postprocess_list import clone
from yolact_b200 import _lib, metrics
from yolact_b200.eval_utils import jaccard, mask_iou, pack_masks
from yolact_b200.metrics import APData, prep_metrics, prep_metrics_list
from yolact_b200.output_utils import _ops_handle, assemble_masks, launch_count, postprocess

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
f32 = np.float32
POISON = 0x7FC0DEAD   # a NaN payload no kernel writes


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def bits_of(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


# ---- the per-image caches, as APData.add computes them --------------------------------------------------------------
def reference_caches(classes, boxes, det_bits, gt, gt_masks, h, w, num_crowd):
    """APData.add's four caches: det_bits [n,h,ceil(w/32)] int32, gt [g,5] relative, gt_masks [g,h,w] host."""
    n, g_all = int(classes.shape[0]), int(gt.shape[0])
    g = g_all - num_crowd
    wpr = (w + 31) // 32
    gb = gt[:, :4].astype(f32)
    gb[:, [0, 2]] *= f32(w)
    gb[:, [1, 3]] *= f32(h)
    gb = cuda(gb) if g_all else torch.zeros(0, 4, device=DEV)
    gbits = (pack_masks(cuda(gt_masks).reshape(g_all, h, w), rows=True).reshape(g_all, h * wpr) if g_all
             else torch.zeros(0, h * wpr, dtype=torch.int32, device=DEV))
    db = det_bits.reshape(n, h * wpr).contiguous()
    miou = lambda b, c: mask_iou(db, b, iscrowd=c, packed=True) if b.shape[0] else torch.empty(n, 0, device=DEV)
    bf = boxes.float()
    return (jaccard(bf, gb[:g]), miou(gbits[:g], False), jaccard(bf, gb[g:], iscrowd=True), miou(gbits[g:], True))


# ---- 1. matching alone on the golden -----------------------------------------------------------------------------------
def _golden_caches(im):
    n, h, w = len(im["classes"]), im["h"], im["w"]
    det_bits = pack_masks(cuda(im["masks"].reshape(n, h, w)), rows=True) if n else None
    if not n:
        return None
    return reference_caches(cuda(im["classes"]), cuda(im["boxes"]), det_bits, im["gt"], im["gt_masks"], h, w,
                            im["num_crowd"])


def _match_items(apd, images, caches):
    """yb_eval_match_list items of images (golden dicts) behind apd's records -> (items, keep_alive, records)."""
    T = len(apd.iou_thresholds)
    items = (_lib.YbEvalMatchItem * len(images))()
    keep, at = [], apd._n
    ptr = lambda t: t.data_ptr() if t is not None and t.numel() else None
    for j, (im, cc) in enumerate(zip(images, caches)):
        n, nc = len(im["classes"]), im["num_crowd"]
        g = im["gt"].reshape(-1, 5).shape[0] - nc
        gt_cls = cuda(im["gt"].reshape(-1, 5)[:, 4].astype(np.int32))
        cls, bs = cuda(im["classes"]).long(), cuda(im["box_scores"])
        ms = cuda(im["mask_scores"]) if im["mask_scores"] is not None else bs
        keep += [gt_cls, cls, bs, ms]
        cc = cc or (None,) * 4
        items[j] = _lib.YbEvalMatchItem(ptr(cc[0]), ptr(cc[1]), ptr(cc[2]), ptr(cc[3]), ptr(cls), ptr(bs), ptr(ms),
                                        ptr(gt_cls[:g]), ptr(gt_cls[g:]), at, n, g, nc)
        at += 2 * T * n
    return items, keep, at - apd._n


def _match_list_call(apd, items, B):
    T = len(apd.iou_thresholds)
    return _lib.load().yb_eval_match_list(_ops_handle(DEV), items, B, apd._thr, T, apd.num_classes,
                                          _lib.ptr(apd._score), _lib.ptr(apd._tag), _lib.ptr(apd._counts),
                                          _lib.ptr(apd._err), _lib.current_stream(DEV))


@pytest.mark.parametrize("chunk", [None, 1, 3, 7])
def test_golden_matching_in_lists(chunk):
    z = _golden()
    ims = golden_images(z)
    caches = [_golden_caches(im) for im in ims]
    apd = APData(int(z["num_classes"]), z["thresholds"].tolist())
    step = chunk or len(ims)
    for s in range(0, len(ims), step):
        items, keep, R = _match_items(apd, ims[s:s + step], caches[s:s + step])
        apd._reserve(R)
        assert _match_list_call(apd, items, len(ims[s:s + step])) == 0
        apd._n += R
    _assert_equal_to(apd, golden_points(z), z["num_gt"], z["ap"], z["nonempty"], golden_all_maps(z))


# ---- 2. from the detections = per image ------------------------------------------------------------------------------
SIZES = [(40, 1), (50, 31), (37, 32), (29, 33), (20, 24), (480, 640), (61, 45), (1080, 1920)]
NONE_AT = 3          # an image without detections in the middle of the list
_state = {}


def net_preds(config):
    if config not in _state:
        net = make_net(config, "f16x3", 256)
        frames = [torch.from_numpy(np.random.RandomState(70 + i).randint(0, 256, s + (3,)).astype(np.uint8)).to(DEV)
                  for i, s in enumerate(SIZES)]
        preds = net.forward_frames(frames)
        preds[NONE_AT] = {"detection": None, "net": preds[NONE_AT]["net"]}
        _state[config] = (net, preds)
    net, preds = _state[config]
    yolact_b200.cfg.replace(net.cfg.copy())
    return preds


def ground_truth(preds, sizes, seed):
    """~7 objects + 1 crowd per image whose masks spill past their boxes; image 1 has g = 0, image 2 only crowds."""
    r = np.random.RandomState(seed)
    gts, gms, ncs = [], [], []
    for i, (h, w) in enumerate(sizes):
        g, nc = (0, 0) if i == 1 else ((0, 2) if i == 2 else (int(r.randint(4, 10)), int(r.randint(0, 3))))
        det = preds[i]["detection"] if i < len(preds) else None
        gt = np.zeros((g + nc, 5), f32)
        c = r.uniform(0, 1, (g + nc, 2))
        wh = r.uniform(0.05, 0.7, (g + nc, 2))
        gt[:, :2], gt[:, 2:4] = c - wh / 2, c + wh / 2
        gt[:, 4] = r.randint(0, 80, g + nc)
        if det is not None and g:   # some ground truth of the detected classes near the detections
            k = min(g, int(det["box"].shape[0]))
            gt[:k, :4] = np.nan_to_num(det["box"][:k].cpu().numpy()) + r.uniform(-0.03, 0.03, (k, 4))
            gt[:k, 4] = det["class"][:k].cpu().numpy()
        gm = np.zeros((g + nc, h, w), f32)
        for j in range(g + nc):
            x1, y1, x2, y2 = gt[j, :4]
            ex = r.uniform(0, 0.1)   # spill past the box
            ys = slice(max(0, int((y1 - ex) * h)), max(1, int(np.ceil((y2 + ex) * h))))
            xs = slice(max(0, int((x1 - ex) * w)), max(1, int(np.ceil((x2 + ex) * w))))
            gm[j, ys, xs] = r.uniform(0, 1, gm[j, ys, xs].shape) < 0.85
        gts.append(gt)
        gms.append(gm if (g + nc) or i % 2 else np.zeros((0, h, w), f32))
        ncs.append(nc)
    return gts, gms, ncs


def per_image_caches(preds, sizes, gts, gms, ncs, crop, thr):
    out = []
    for i, (h, w) in enumerate(sizes):
        classes, _, boxes, masks = postprocess(clone(preds), w, h, i, crop_masks=crop, score_threshold=thr,
                                               mask_format="bits")
        if classes.size(0) == 0:
            continue
        out.append((i,) + reference_caches(classes, boxes, masks, gts[i], gms[i], h, w, ncs[i]))
    return out


def assert_caches_equal(lst, want):
    assert [im[0] for im in lst.images] == [wnt[0] for wnt in want]
    for im, wnt in zip(lst.images, want):
        for a, b in zip(im[4:], wnt[1:]):
            assert tuple(a.shape) == tuple(b.shape)
            assert np.array_equal(bits_of(a), bits_of(b)), (im[:4], np.argwhere(bits_of(a) != bits_of(b))[:5])


def records(apd):
    score, tag = apd._host_records()
    return score.view(np.uint32), tag


def assert_same_apdata(a, b):
    sa, ta = records(a)
    sb, tb = records(b)
    assert a.num_records == b.num_records and np.array_equal(sa, sb) and np.array_equal(ta, tb)
    assert np.array_equal(a.num_gt_positives(), b.num_gt_positives())
    (pa, na), (pb, nb) = a.get_ap(), b.get_ap()
    assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64)) and np.array_equal(na, nb)


def per_image_apdata(preds, sizes, gts, gms, ncs, crop, thr, images=None):
    apd = APData(80)
    for i in (range(len(sizes)) if images is None else images):
        h, w = sizes[i]
        prep_metrics(apd, clone(preds)[i:i + 1], None, gts[i], gms[i], h, w, ncs[i], i, crop_masks=crop,
                     score_threshold=thr)
    return apd


@pytest.mark.parametrize("config", ["yolact_base_config", "yolact_plus_resnet50_config"])
@pytest.mark.parametrize("crop", [True, False])
@pytest.mark.parametrize("thr", [0.0, 0.15])
def test_list_equals_per_image(config, crop, thr):
    preds = net_preds(config)
    gts, gms, ncs = ground_truth(preds, SIZES, 5)
    want = per_image_caches(preds, SIZES, gts, gms, ncs, crop, thr)
    assert len(want) >= (4 if thr == 0 else 1)
    lst = metrics._iou_list(80, DEV, clone(preds), SIZES, gts, gms, ncs, crop, thr)
    assert_caches_equal(lst, want)
    a = per_image_apdata(preds, SIZES, gts, gms, ncs, crop, thr)
    b = APData(80)
    prep_metrics_list(b, clone(preds), SIZES, gts, gms, ncs, crop_masks=crop, score_threshold=thr)
    assert b.num_records > 0
    assert_same_apdata(a, b)
    if config == "yolact_plus_resnet50_config":   # YOLACT++'s [box, mask] scores reach the records
        assert any(isinstance(postprocess(clone(preds), w, h, i)[1], list) for i, (h, w) in enumerate(SIZES)
                   if preds[i]["detection"] is not None)


def test_ground_truth_on_the_device_and_as_uint8():
    preds = net_preds("yolact_base_config")
    gts, gms, ncs = ground_truth(preds, SIZES, 8)
    a = per_image_apdata(preds, SIZES, gts, gms, ncs, True, 0.0)
    mixed = [cuda(m) if i % 3 == 0 else (m.astype(np.uint8) if i % 3 == 1 else m.astype(np.float64))
             for i, m in enumerate(gms)]
    b = APData(80)
    prep_metrics_list(b, clone(preds), SIZES, gts, mixed, ncs)
    assert_same_apdata(a, b)


# ---- 3. adversarial boxes -----------------------------------------------------------------------------------------------
def test_adversarial_boxes():
    preds = net_preds("yolact_base_config")
    bad = clone(preds)
    adversarial = [[np.nan, 0.1, 0.5, 0.5], [0.7, 0.1, 0.2, 0.6], [0.3, 0.2, 0.3, 0.8], [-0.1, -0.1, 1.1, 1.1],
                   [1.2, 1.3, 1.5, 1.6], [0.1, np.nan, np.nan, 0.9]]
    for p in bad:
        if p["detection"] is not None:
            k = min(len(adversarial), int(p["detection"]["box"].shape[0]))
            p["detection"]["box"][:k] = torch.tensor(adversarial[:k], device=DEV)
    gts, gms, ncs = ground_truth(bad, SIZES, 9)
    for crop in (True, False):
        want = per_image_caches(bad, SIZES, gts, gms, ncs, crop, 0.0)
        assert_caches_equal(metrics._iou_list(80, DEV, clone(bad), SIZES, gts, gms, ncs, crop, 0.0), want)
        assert any(np.isnan(w[2].cpu().numpy()).any() or np.isnan(w[1].cpu().numpy()).any() for w in want)
        assert_same_apdata(per_image_apdata(bad, SIZES, gts, gms, ncs, crop, 0.0),
                           _list_apdata(bad, SIZES, gts, gms, ncs, crop))


def _list_apdata(preds, sizes, gts, gms, ncs, crop=True, thr=0.0):
    apd = APData(80)
    prep_metrics_list(apd, clone(preds), sizes, gts, gms, ncs, crop_masks=crop, score_threshold=thr)
    return apd


# ---- 4. every output written, nothing else; 6. one launch per list ---------------------------------------------------------
GUARD = 37


def synthetic_iou_case(specs, seed):
    """specs: (n, h, w, g_all, num_crowd) per image on one prototype map -> the images' device inputs, pixel boxes and
    bit masks (from yb_postprocess), and ground truth."""
    ph, pw, k = 36, 52, 32
    out = []
    for i, (n, h, w, g_all, nc) in enumerate(specs):
        proto, coef, box = ME.random_case(seed + i, n, ph, pw, k)
        if n > 2:
            box[1] = [-0.1, -0.1, 1.1, 1.1]
            box[2] = [0.4, np.nan, 0.6, 0.7]
        tp, tc, tb = cuda(proto), cuda(coef.reshape(n, k)), cuda(box.reshape(n, 4))
        masks, px, _ = assemble_masks(tp, tc, tb, h, w, True, "bits")
        r = np.random.RandomState(seed + 100 + i)
        gt = np.concatenate([np.sort(r.uniform(0, 1, (g_all, 4)), 1)[:, [0, 1, 2, 3]],
                             r.randint(0, 80, (g_all, 1))], 1).astype(f32)
        gm = (r.uniform(0, 1, (g_all, h, w)) < 0.4).astype(f32)
        out.append(dict(proto=tp, coef=tc, box=tb, px=px, masks=masks, gt=gt, gm=gm, n=n, h=h, w=w, g_all=g_all,
                        nc=nc))
    return out, (ph, pw, k)


def iou_items(case, caches_at):
    """yb_eval_iou_list items; caches_at(j, which, rows, cols) -> the device tensor for that output."""
    items = (_lib.YbEvalIouItem * len(case))()
    keep = []
    for j, c in enumerate(case):
        im = metrics._gt_image(c["gt"], c["gm"], c["h"], c["w"], c["nc"], 80, "t")
        wpr = (c["w"] + 31) // 32
        gb = cuda(im.boxes) if im.g_all else None
        bits = pack_masks(cuda(c["gm"]), rows=True) if im.g_all else None
        g = im.g_all - c["nc"]
        outs = [caches_at(j, q, c["n"], (g, g, c["nc"], c["nc"])[q]) for q in range(4)]
        keep += [gb, bits] + outs
        p = lambda t: t.data_ptr() if t is not None and t.numel() else None
        items[j] = _lib.YbEvalIouItem(c["proto"].data_ptr(), p(c["coef"]), p(c["box"]), p(c["px"]), p(bits), p(gb),
                                      *[p(o) for o in outs], c["n"], c["h"], c["w"], im.g_all, c["nc"])
        assert wpr * 32 >= c["w"]
    return items, keep


SPECS = [(5, 33, 47, 6, 2), (0, 20, 20, 3, 1), (4, 1, 1, 2, 0), (3, 64, 31, 0, 0), (6, 17, 100, 3, 3), (7, 128, 96, 9, 1),
         (2, 5, 33, 4, 0), (1, 300, 1250, 2, 1)]


def test_every_cache_written_nothing_else_and_one_launch():
    case, (ph, pw, k) = synthetic_iou_case(SPECS, 21)
    sizes = [(c["n"], (c["g_all"] - c["nc"], c["g_all"] - c["nc"], c["nc"], c["nc"])) for c in case]
    total = sum(n * m for n, ms in sizes for m in ms)
    buf = torch.full((total + GUARD * (4 * len(case) + 1),), POISON, dtype=torch.int32, device=DEV)
    at = {}
    off = GUARD

    def caches_at(j, q, n, m):
        nonlocal off
        t = buf[off:off + n * m].view(torch.float32).view(n, m)
        at[(j, q)] = (off, n * m)
        off += n * m + GUARD
        return t
    items, keep = iou_items(case, caches_at)
    lib = _lib.load()
    h = _ops_handle(DEV, k)
    before = launch_count()
    assert lib.yb_eval_iou_list(h, items, len(case), ph, pw, k, 1, _lib.current_stream(DEV)) == 0
    assert launch_count() - before == 1
    host = buf.cpu().numpy()
    written = np.zeros(len(host), bool)
    for j, c in enumerate(case):
        want = reference_caches(torch.zeros(c["n"]), c["px"], c["masks"], c["gt"], c["gm"], c["h"], c["w"], c["nc"]) \
            if c["n"] else [torch.empty(0, m) for m in sizes[j][1]]
        for q in range(4):
            o, ln = at[(j, q)]
            written[o:o + ln] = True
            assert np.array_equal(host[o:o + ln], bits_of(want[q]).reshape(-1)), (j, q)
    assert (host[~written] == POISON).all()
    for B in (1, 3, len(case)):   # one launch whatever the list length
        before = launch_count()
        assert lib.yb_eval_iou_list(h, items, B, ph, pw, k, 1, _lib.current_stream(DEV)) == 0
        assert launch_count() - before == 1
    assert np.array_equal(buf.cpu().numpy(), host)   # repeated calls: the same bits


def test_every_record_written_nothing_else_and_one_launch():
    z = _golden()
    ims = golden_images(z)[:9]
    caches = [_golden_caches(im) for im in ims]
    apd = APData(int(z["num_classes"]), z["thresholds"].tolist())
    T = len(apd.iou_thresholds)
    # the images' slots with a guard band after each
    items, keep, R = _match_items(apd, ims, caches)
    at = GUARD
    for j, im in enumerate(ims):
        items[j].rec_offset = at
        at += 2 * T * len(im["classes"]) + GUARD
    apd._reserve(at)
    apd._score.view(torch.int32).fill_(POISON)
    apd._tag.fill_(-7)
    before = launch_count()
    assert _match_list_call(apd, items, len(ims)) == 0
    assert launch_count() - before == 1
    score, tag = apd._score.view(torch.int32).cpu().numpy(), apd._tag.cpu().numpy()
    slot = np.zeros(len(score), bool)
    for j, im in enumerate(ims):
        o = items[j].rec_offset
        slot[o:o + 2 * T * len(im["classes"])] = True
    assert (score[slot] != POISON).all() and (tag[slot] != -7).all()
    assert (score[~slot] == POISON).all() and (tag[~slot] == -7).all()
    # the slots hold what yb_eval_match writes per image
    ref = APData(int(z["num_classes"]), z["thresholds"].tolist())
    from tests.test_gpu_map import _add
    for im in ims:
        _add(ref, im, "f32")
    rs, rt = ref._host_records()
    assert np.array_equal(score[slot], rs.view(np.int32)) and np.array_equal(tag[slot], rt)
    assert np.array_equal(apd.num_gt_positives(), ref.num_gt_positives())


def test_prep_metrics_list_launches_do_not_grow_with_the_list():
    preds = net_preds("yolact_base_config")
    gts, gms, ncs = ground_truth(preds, SIZES, 5)
    live = [i for i, p in enumerate(preds) if p["detection"] is not None and len(gts[i])]
    counts = []
    for sel in (live[:1], live):
        apd = APData(80)
        before = launch_count()
        prep_metrics_list(apd, [clone(preds)[i] for i in sel], [SIZES[i] for i in sel], [gts[i] for i in sel],
                          [gms[i] for i in sel], [ncs[i] for i in sel])
        counts.append(launch_count() - before)
    assert len(live) >= 3 and counts[0] == counts[1], counts


def test_no_host_sync_at_threshold_zero():
    preds = net_preds("yolact_base_config")
    gts, gms, ncs = ground_truth(preds, SIZES, 5)
    apd = APData(80)
    prep_metrics_list(apd, clone(preds), SIZES, gts, gms, ncs)   # first call: handles, buffers
    p = clone(preds)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        prep_metrics_list(apd, p, SIZES, gts, gms, ncs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert apd.num_records > 0


# ---- 5. refusals ----------------------------------------------------------------------------------------------------------
def test_c_abi_refusals():
    case, (ph, pw, k) = synthetic_iou_case([(3, 20, 40, 3, 1)], 4)
    outs = {}

    def caches_at(j, q, n, m):
        outs[q] = torch.full((n, m), 7.0, device=DEV)
        return outs[q]
    items, keep = iou_items(case, caches_at)
    lib = _lib.load()
    h = _ops_handle(DEV, k)
    host = torch.zeros(64)
    good = _lib.YbEvalIouItem.from_buffer_copy(items[0])

    def iou(B=1, kk=k, **kw):
        it = (_lib.YbEvalIouItem * 1)()
        it[0] = _lib.YbEvalIouItem.from_buffer_copy(good)
        for f, v in kw.items():
            setattr(it[0], f, v)
        return lib.yb_eval_iou_list(h, it, B, ph, pw, kk, 1, _lib.current_stream(DEV))
    bad = [dict(n=1025), dict(n=-1), dict(out_h=0), dict(out_w=-1), dict(num_crowd=4), dict(num_crowd=-1),
           dict(g_all=1025 + 1, num_crowd=1), dict(g_all=2050, num_crowd=1025), dict(proto=None), dict(coef=None),
           dict(box=None), dict(boxes_px=None), dict(gt_bits=None), dict(gt_boxes=None), dict(box_iou=None),
           dict(mask_iou=None), dict(crowd_box_iou=None), dict(crowd_mask_iou=None), dict(gt_bits=host.data_ptr()),
           dict(box_iou=host.data_ptr()), dict(proto=host.data_ptr()), dict(B=-1), dict(B=70000), dict(kk=6),
           dict(kk=132)]
    for kw in bad:
        assert iou(**kw) == -1, kw   # YB_ERR_INVALID
    torch.cuda.synchronize()
    assert all((o == 7.0).all() for o in outs.values())
    assert iou() == 0 and iou(B=0) == 0 and iou(n=0, proto=None, coef=None, box=None, boxes_px=None) == 0

    # yb_eval_match_list
    z = _golden()
    im = [x for x in golden_images(z) if len(x["classes"]) and x["num_crowd"] and
          x["gt"].reshape(-1, 5).shape[0] > x["num_crowd"]][0]
    apd = APData(80)
    its, keep2, R = _match_items(apd, [im], [_golden_caches(im)])
    apd._reserve(R)
    apd._score.fill_(3.0)
    apd._counts.fill_(5)
    good_m = _lib.YbEvalMatchItem.from_buffer_copy(its[0])

    def match(B=1, T=10, C=80, rec=apd._score, **kw):
        it = (_lib.YbEvalMatchItem * 1)()
        it[0] = _lib.YbEvalMatchItem.from_buffer_copy(good_m)
        for f, v in kw.items():
            setattr(it[0], f, v)
        thr = (ctypes.c_double * 32)(*([0.5] * 32))
        return lib.yb_eval_match_list(_ops_handle(DEV), it, B, thr, T, C, _lib.ptr(rec), _lib.ptr(apd._tag),
                                      _lib.ptr(apd._counts), _lib.ptr(apd._err), _lib.current_stream(DEV))
    bad = [dict(n=1025), dict(g=1025), dict(num_crowd=1025), dict(n=-1), dict(T=0), dict(T=33), dict(C=0),
           dict(C=2049), dict(rec_offset=-1), dict(cls=None), dict(box_score=None), dict(mask_score=None),
           dict(box_iou=None), dict(mask_iou=None), dict(gt_cls=None), dict(crowd_box_iou=None),
           dict(crowd_mask_iou=None), dict(crowd_cls=None), dict(cls=host.data_ptr()), dict(mask_iou=host.data_ptr()),
           dict(rec=host), dict(B=-1)]
    for kw in bad:
        assert match(**kw) == -1, kw
    torch.cuda.synchronize()
    assert (apd._score == 3.0).all() and (apd._counts == 5).all()
    assert match() == 0 and match(B=0) == 0


def test_python_refusals():
    preds = net_preds("yolact_base_config")
    gts, gms, ncs = ground_truth(preds, SIZES, 5)
    apd = APData(80)
    i0 = [i for i, p in enumerate(preds) if p["detection"] is not None and len(gts[i]) > ncs[i] and i > 2][0]
    cases = [dict(sizes=SIZES[:-1]), dict(gts=gts[:-1]), dict(gms=gms[:-1]), dict(ncs=ncs[:-1])]
    bad_cls = [g.copy() for g in gts]
    bad_cls[i0][0, 4] = 80
    cases.append(dict(gts=bad_cls))
    bad_nc = list(ncs)
    bad_nc[i0] = len(gts[i0]) + 1
    cases.append(dict(ncs=bad_nc))
    bad_nc2 = list(ncs)
    bad_nc2[i0] = -1
    cases.append(dict(ncs=bad_nc2))
    bad_gm = list(gms)
    bad_gm[i0] = gms[i0][:, :-1]
    cases.append(dict(gms=bad_gm))
    for kw in cases:
        with pytest.raises(ValueError):
            prep_metrics_list(apd, clone(preds), kw.get("sizes", SIZES), kw.get("gts", gts), kw.get("gms", gms),
                              kw.get("ncs", ncs))
    no_proto = clone(preds)
    del no_proto[i0]["detection"]["proto"]
    with pytest.raises(ValueError):
        prep_metrics_list(apd, no_proto, SIZES, gts, gms, ncs)
    save = yolact_b200.cfg.eval_mask_branch
    yolact_b200.cfg.eval_mask_branch = False
    try:
        with pytest.raises(ValueError, match="eval_mask_branch"):
            prep_metrics_list(apd, clone(preds), SIZES, gts, gms, ncs)
    finally:
        yolact_b200.cfg.eval_mask_branch = save
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            prep_metrics_list(APData(80, device="cuda:1"), clone(preds), SIZES, gts, gms, ncs)
    else:   # an accumulator on another device: the check compares devices before anything runs
        other = APData(80)
        other._device = torch.device("cuda", 7)
        with pytest.raises(ValueError):
            prep_metrics_list(other, clone(preds), SIZES, gts, gms, ncs)
    assert apd.num_records == 0 and int(apd._counts.sum()) == 0


# ---- 7. mixing calls --------------------------------------------------------------------------------------------------------
def test_mixing_per_image_and_list_calls():
    preds = net_preds("yolact_plus_resnet50_config")
    gts, gms, ncs = ground_truth(preds, SIZES, 12)
    a = per_image_apdata(preds, SIZES, gts, gms, ncs, True, 0.0)
    b = APData(80)
    p = clone(preds)
    for i in (0, 1):
        prep_metrics(b, p[i:i + 1], None, gts[i], gms[i], SIZES[i][0], SIZES[i][1], ncs[i], i)
    prep_metrics_list(b, p[2:6], SIZES[2:6], gts[2:6], gms[2:6], ncs[2:6])
    prep_metrics(b, p[6:7], None, gts[6], gms[6], SIZES[6][0], SIZES[6][1], ncs[6], 6)
    prep_metrics_list(b, p[7:], SIZES[7:], gts[7:], gms[7:], ncs[7:])
    assert_same_apdata(a, b)
