"""--output_coco_json on the GPU: yb_coco_rle_list's strings, written straight from the detections, against the strings
of the materialised masks (postprocess(mask_format='bits') + mask_run_lengths + rle_to_string), row for row, at the
crop, value, resize and layout edges of tests/test_gpu_mask_edges.py; the arena retry; Detections over lists, through
the network and on the golden; install_coco_json; and the C ABI's refusals."""
import ctypes
import types

import numpy as np
import pytest
import torch

import yolact_b200
from oracle.eval_oracle import rle_decode, rle_from_string
from tests import test_gpu_mask_edges as ME
from tests.test_coco_json_host import category_table, golden, golden_images
from tests.helpers import cfg_for
from tests.test_gpu_frames import make_net
from tests.test_gpu_postprocess_list import clone
from yolact_b200 import _lib
from yolact_b200.eval_utils import encode_masks, mask_run_lengths, rle_to_string
from yolact_b200.metrics import Detections, append_coco_records, coco_rle_list
from yolact_b200.output_utils import _ops_handle, assemble_masks, postprocess, unpack_bits

pytestmark = pytest.mark.gpu
f32 = np.float32
DEV = torch.device("cuda")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def list_strings(cases, crop=True, cap=None):
    """cases: (proto, coef, box, h, w) with one prototype shape -> (strings per image, calls)."""
    ph, pw, k = cases[0][0].shape
    keep, items = [], (_lib.YbPostItem * len(cases))()
    for i, (proto, coef, box, h, w) in enumerate(cases):
        n = len(box)
        tp, tc, tb = cuda(np.asarray(proto, f32)), cuda(np.asarray(coef, f32).reshape(n, k)), cuda(
            np.asarray(box, f32).reshape(n, 4))
        keep += [tp, tc, tb]
        items[i] = _lib.YbPostItem(tp.data_ptr(), tc.data_ptr() or None, tb.data_ptr() or None, None, None, None, n,
                                   h, w)
    rows = sum(len(c[2]) for c in cases)
    strings, _, calls = coco_rle_list(items, rows, ph, pw, k, crop, cap=cap)
    out, r = [], 0
    for c in cases:
        out.append(strings[r:r + len(c[2])])
        r += len(c[2])
    return out, calls


def materialised_strings(proto, coef, box, h, w, crop=True, decode=True):
    n = len(box)
    if n == 0:
        return []
    masks, _, _ = assemble_masks(cuda(np.asarray(proto, f32)), cuda(np.asarray(coef, f32)), cuda(np.asarray(box, f32)),
                                 h, w, crop, "bits")
    runs = mask_run_lengths(masks, "bits", w)
    strings = [rle_to_string(r).decode("ascii") for r in runs]
    if decode and h * w <= 600 * 600:
        px = unpack_bits(masks, w).cpu().numpy()
        for i in range(min(n, 4)):
            assert (rle_decode(rle_from_string(strings[i].encode()), h, w) == px[i]).all()
    return strings


def check_cases(cases, crop=True):
    got, calls = list_strings(cases, crop)
    for (proto, coef, box, h, w), g in zip(cases, got):
        want = materialised_strings(proto, coef, box, h, w, crop)
        assert len(g) == len(want)
        for i, (a, b) in enumerate(zip(g, want)):
            assert a == b, "%dx%d<-%s crop=%d row %d: %r != %r" % (h, w, proto.shape, crop, i, a[:40], b[:40])
    return calls


# ---- 1. strings from the detections = strings of the materialised masks ---------------------------------------------
@pytest.mark.parametrize("ph,pw,h,w", [(36, 52, 148, 204), (138, 138, 550, 550), (36, 52, 28, 44), (48, 40, 144, 136)])
@pytest.mark.parametrize("crop", [True, False])
def test_crop_geometry(ph, pw, h, w, crop):
    box = ME.geometry_boxes(ph, pw)
    proto, coef = ME.saturated(ph + pw + h, len(box), ph, pw)
    check_cases([(proto, coef, box, h, w)], crop)


@pytest.mark.parametrize("ph,pw,h,w,k", [(138, 138, 550, 550, 32), (48, 40, 203, 277, 4), (36, 52, 64, 96, 128),
                                         (138, 138, 101, 83, 4)])
def test_ramp_and_checkerboard(ph, pw, h, w, k):
    proto, coef, box = ME.ramp_case(h + w, 10, ph, pw, k)
    check_cases([(proto, coef, box, h, w)])
    proto, coef, box = ME.checker_case(6, ph, pw, k)
    for crop in (True, False):
        check_cases([(proto, coef, box, h, w)], crop)


@pytest.mark.parametrize("ph,pw,k,h,w,n", ME.RESIZE)
def test_resize_ratios(ph, pw, k, h, w, n):
    proto, coef, box = ME.random_case(ph * 7 + pw + h * 3 + w, n, ph, pw, k, 0.8 if k < 128 else 0.4)
    box[0] = [-0.1, -0.1, 1.1, 1.1]   # one mask over the whole frame
    check_cases([(proto, coef, box, h, w)])


@pytest.mark.parametrize("crop", [True, False])
@pytest.mark.parametrize("ph,pw,h,w", [(138, 138, 550, 550), (48, 40, 203, 277)])
def test_nonfinite_boxes(crop, ph, pw, h, w):
    box = ME.nonfinite_boxes()
    proto, coef = ME.saturated(11, len(box), ph, pw)
    check_cases([(proto, coef, box, h, w)], crop)


def test_wide_frames_take_several_column_chunks():
    proto, coef, box = ME.random_case(5, 4, 138, 138, 32)
    box[0] = [-0.1, -0.1, 1.1, 1.1]
    check_cases([(proto, coef, box, 8, 3000), (proto, coef, box, 2, 9000)])


def test_list_mixing_sizes_and_empty_images():
    ph, pw, k = 138, 138, 32
    cases = []
    for i, (n, h, w) in enumerate(ME.LIST_SIZES + [(3, 2208, 1242)]):
        proto, coef, box = ME.random_case(500 + i, n, ph, pw, k)
        cases.append((proto, coef, box, h, w))
    cases[3][2][1] = [0.1, 0.2, np.nan, np.inf]
    for crop in (True, False):
        check_cases(cases, crop)
    got, _ = list_strings(cases[1:2])   # only an n = 0 image
    assert got == [[]]


# ---- 2. the arena retry ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap", [0, 4, (10 ** 6, 3), (5, 10 ** 6)])
def test_small_arena_retries_once(cap):
    proto, coef, box = ME.checker_case(6, 48, 40, 4)
    cases = [(proto, coef, box, 208, 280), (proto, coef[:2], box[:2], 33, 17)]
    want, calls = list_strings(cases, cap=10 ** 7)
    assert calls == 1
    got, calls = list_strings(cases, cap=cap)
    assert calls == 2 and got == want


# ---- 3. Detections: a list = one call per image --------------------------------------------------------------------------
def synthetic_preds(sizes, seed):
    yolact_b200.cfg.replace(cfg_for("yolact_base_config").copy())   # no maskiou_net: the rows need no net
    preds = []
    for i, (h, w) in enumerate(sizes):
        n = (seed + i) % 5 * 3
        proto, coef, box = ME.random_case(seed + i, n, 69, 69, 32)
        det = {"box": cuda(box), "mask": cuda(coef), "class": torch.arange(n, device=DEV) * 7 % 80,
               "score": torch.linspace(0.9, 0.1, n, device=DEV), "proto": cuda(proto)}
        preds.append({"net": None, "detection": det if n else None})
    return preds


def test_list_equals_per_image():
    sizes = [(60, 80), (1, 1), (277, 203), (33, 600), (480, 640), (17, 9)]
    table = list(range(1, 81))
    whole, single = Detections(table), Detections(table)
    whole.add(synthetic_preds(sizes, 3), sizes, [10 * i + 1 for i in range(len(sizes))])
    for i, p in enumerate(synthetic_preds(sizes, 3)):
        single.add([p], [sizes[i]], [10 * i + 1])
    assert whole.bbox_data == single.bbox_data and whole.mask_data == single.mask_data
    assert len(whole.mask_data) > 10


# ---- 4. through the network ---------------------------------------------------------------------------------------------
def route_a(dets, preds, sizes, image_ids, crop_masks=True, score_threshold=0):
    """Today's best route: postprocess(mask_format='bits') + encode_masks + the records, per image."""
    for p, (h, w), image_id in zip(preds, sizes, image_ids):
        classes, scores, boxes, masks = postprocess([p], w, h, crop_masks=crop_masks, score_threshold=score_threshold,
                                                    mask_format="bits")
        if classes.size(0) == 0:
            continue
        bs, ms = (scores[0], scores[1]) if isinstance(scores, list) else (scores, scores)
        counts = [e["counts"].decode("ascii") for e in encode_masks(masks, "bits", w)]
        append_coco_records(dets.bbox_data, dets.mask_data, dets.category_of, image_id, classes.cpu().numpy(),
                            boxes.cpu().numpy(), bs.cpu().numpy(), ms.cpu().numpy(), counts, h, w)


def dumped(dets, tmp_path, tag):
    b, m = tmp_path / ("%s_bbox.json" % tag), tmp_path / ("%s_mask.json" % tag)
    dets.dump(str(b), str(m))
    return b.read_bytes(), m.read_bytes()


@pytest.mark.parametrize("config", ["yolact_base_config", "yolact_plus_resnet50_config"])
@pytest.mark.parametrize("size", [(480, 640), (550, 550)])
def test_through_the_network(config, size, tmp_path):
    net = make_net(config, "f16x3", 550)
    sizes = [size] * 3
    preds = net.forward_frames([torch.from_numpy(np.random.RandomState(40 + i).randint(0, 256, size + (3,)).astype(
        np.uint8)).cuda() for i in range(3)])
    thr_mid = float(preds[0]["detection"]["score"].median()) if preds[0]["detection"] is not None else 0.15
    for thr in (0, 0.15, thr_mid):
        table = list(range(100, 180))
        a, b = Detections(table), Detections(table)
        route_a(a, clone(preds), sizes, [5, 9, 2], score_threshold=thr)
        b.add(clone(preds), sizes, [5, 9, 2], score_threshold=thr)
        assert dumped(a, tmp_path, "a") == dumped(b, tmp_path, "b")
        if thr == 0:
            assert len(b.mask_data) > 0
            if net.cfg.use_maskiou and getattr(net.cfg, "rescore_mask", False) and not net.cfg.rescore_bbox:
                assert any(x["score"] != y["score"] for x, y in zip(b.bbox_data, b.mask_data))


# ---- 5. the golden --------------------------------------------------------------------------------------------------------
def test_golden_on_the_gpu(tmp_path):
    z = golden()
    dets = Detections(category_table(z))
    for im in golden_images(z):
        counts = [e["counts"].decode("ascii") for e in encode_masks(cuda(im["masks"]), "u8")]
        ms = im["mask_scores"] if im["mask_scores"] is not None else im["scores"]
        append_coco_records(dets.bbox_data, dets.mask_data, dets.category_of, im["image_id"], im["classes"],
                            im["boxes"], im["scores"], ms, counts, im["h"], im["w"])
    assert dumped(dets, tmp_path, "g") == (z["bbox_json"].tobytes(), z["mask_json"].tobytes())


# ---- 6. integration -------------------------------------------------------------------------------------------------------
class RefDetections:
    def __init__(self):
        self.bbox_data, self.mask_data = [], []


def stand_in_eval(calls):
    E = types.ModuleType("eval")
    E.args = types.SimpleNamespace(output_coco_json=True, crop=True, score_threshold=0)
    E.cfg = types.SimpleNamespace(dataset=types.SimpleNamespace(class_names=["c%d" % i for i in range(80)]))
    E.iou_thresholds = [x / 100 for x in range(50, 100, 5)]
    E.get_coco_cat = lambda c: 1000 + c
    E.prep_metrics = lambda *a, **k: calls.append("prep")
    E.calc_map = lambda ap_data: "original"
    E.postprocess = postprocess
    return E


@pytest.mark.parametrize("order", ["coco_only", "coco_then_metrics", "metrics_then_coco"])
def test_install_coco_json(order):
    from integration.use_b200 import install_coco_json, install_metrics
    calls = []
    E = stand_in_eval(calls)
    if order == "metrics_then_coco":
        install_metrics(E)
    install_coco_json(E)
    if order == "coco_then_metrics":
        install_metrics(E)
    sizes = [(60, 80), (277, 203), (33, 600)]
    preds = synthetic_preds(sizes, 4)
    got, want = RefDetections(), Detections(E.get_coco_cat)
    for i, (p, (h, w)) in enumerate(zip(preds, sizes)):
        E.prep_metrics({}, [p], None, None, None, h, w, 0, 100 + i, got)
    route_a(want, synthetic_preds(sizes, 4), sizes, [100, 101, 102])
    assert got.bbox_data == want.bbox_data and got.mask_data == want.mask_data and got.mask_data
    assert calls == []
    E.args.output_coco_json = False
    if order == "coco_only":
        E.prep_metrics({}, [preds[0]], None, None, None, 60, 80, 0, 0, got)
        assert calls == ["prep"]


def test_detect_mode_is_refused():
    preds = synthetic_preds([(20, 20)], 1)
    save = yolact_b200.cfg.eval_mask_branch
    yolact_b200.cfg.eval_mask_branch = False
    try:
        with pytest.raises(ValueError, match="eval_mask_branch"):
            Detections(list(range(80))).add(preds, [(20, 20)], [0])
    finally:
        yolact_b200.cfg.eval_mask_branch = save


# ---- 7. C ABI refusals ----------------------------------------------------------------------------------------------------
def test_c_abi_refusals():
    lib = _lib.load()
    ph, pw, k = 16, 16, 4
    proto, coef, box = cuda(np.ones((ph, pw, k), f32)), cuda(np.ones((2, k), f32)), cuda(np.full((2, 4), 0.5, f32))
    box[:, 2:] = 0.9
    runs = torch.full((64,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    chars = torch.full((64,), 0xA5, dtype=torch.uint8, device=DEV)
    off = torch.full((4,), -3, dtype=torch.int64, device=DEV)
    ln = torch.full((4,), -3, dtype=torch.int32, device=DEV)
    need = torch.full((2,), -3, dtype=torch.int64, device=DEV)
    host = torch.zeros(8)
    outs = [runs, chars, off, ln, need]
    snap = [t.clone() for t in outs]
    h = _ops_handle(DEV, k)

    def call(item=None, runs_p=runs, runs_cap=64, chars_p=chars, chars_cap=64, off_p=off, len_p=ln, need_p=need, B=1):
        items = (_lib.YbPostItem * 1)()
        items[0] = item or _lib.YbPostItem(proto.data_ptr(), coef.data_ptr(), box.data_ptr(), None, None, None, 2, 20, 20)
        ptr = lambda t: None if t is None else t.data_ptr()
        return lib.yb_coco_rle_list(h, items, B, ph, pw, k, 1, ptr(runs_p), runs_cap, ptr(chars_p), chars_cap,
                                    ptr(off_p), ptr(len_p), ptr(need_p), _lib.current_stream(DEV))

    item = lambda **kw: _lib.YbPostItem(**{**dict(proto=proto.data_ptr(), coef=coef.data_ptr(), box=box.data_ptr(),
                                                  n=2, out_h=20, out_w=20), **kw})
    bad = [dict(item=item(proto=None)), dict(item=item(coef=None)), dict(item=item(box=None)), dict(item=item(n=-1)),
           dict(item=item(out_h=0)), dict(item=item(out_w=-5)), dict(runs_p=None), dict(chars_p=None),
           dict(off_p=None), dict(len_p=None), dict(need_p=None), dict(runs_cap=-1), dict(chars_cap=-1),
           dict(item=item(proto=host.data_ptr())), dict(item=item(box=host.data_ptr())), dict(chars_p=host),
           dict(need_p=host), dict(B=-1)]
    for kw in bad:
        assert call(**kw) == -1, kw   # YB_ERR_INVALID
    torch.cuda.synchronize()
    for t, s in zip(outs, snap):
        assert torch.equal(t, s)
    assert call() == 0 and call(B=0) == 0 and call(item=item(n=0, proto=None, coef=None, box=None)) == 0
    torch.cuda.synchronize()
    assert need.tolist() == [0, 0]
