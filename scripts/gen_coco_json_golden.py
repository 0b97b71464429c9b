"""Generates tests/golden/coco_json_unit.npz: eval.py's --output_coco_json records, written by the REAL reference on the
CPU.

    python scripts/gen_coco_json_golden.py      # needs the reference checkout at oracle/gen_golden.py's REF

Runs the reference's own prep_metrics with --output_coco_json (eval.py:386-429), Detections.add_bbox / add_mask
(:303-330), prep_coco_cats (:283-288) and Detections.dump (:332-340) into a temporary directory.  Shims, never edits to
the reference: oracle/gen_golden.py's install_shims, `torch.Tensor.cuda` as the identity, eval.postprocess replaced by a
stub that returns the image's stored (classes, scores -- a tensor or YOLACT++'s [box, mask] list --, int64 pixel boxes,
0/1 masks), and pycocotools.mask.encode set to the oracle's restatement (oracle/eval_oracle.py rle_counts +
rle_to_string, returning bytes as pycocotools does).  The RLE string itself stays restated, not pinned to pycocotools;
everything around it is the reference's.

The images cover zero-area pixel boxes (x1 == x2, y1 == y2: skipped), empty and full masks (a set first pixel gives a
leading 0 run), a mask whose last pixel is set, a 1 x 1 image, classes 0 and 79, fp32 scores with long reprs, YOLACT++
[box, mask] score lists, image ids that are not 0..N, and a seeded random batch.

Stored: per image `img{i}_*` (h, w, image_id, classes, scores, optional mask_scores, boxes, masks bit-packed along the
last axis), `coco_cats_keys` / `coco_cats_values` (the reference's class index -> category id table after
prep_coco_cats), and the two JSON files' bytes (`bbox_json`, `mask_json`).
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def crafted_images():
    imgs = []
    h, w = 24, 32
    m = np.zeros((5, h, w), np.uint8)
    m[1] = 1                                   # full: leading 0 run
    m[2, 3:9, 4:20] = 1
    m[3, h - 1, w - 1] = 1                     # the last pixel
    m[4, 0, 0] = 1                             # the first pixel only
    boxes = np.array([[4, 4, 4, 10],           # zero width: skipped
                      [0, 0, w, h], [4, 3, 20, 9], [31, 23, 32, 24], [0, 0, 1, 1]], np.int64)
    scores = np.array([0.9, 0.8123456789, 1 / 3, 0.1 + 0.2, 2 / 7], np.float32)
    imgs.append(dict(h=h, w=w, image_id=139, classes=np.array([3, 0, 79, 40, 1]), scores=scores, boxes=boxes, masks=m))
    # empty masks with a positive box area, and a zero-height box
    m = np.zeros((3, 16, 16), np.uint8)
    m[2, 5:7, 5:7] = 1
    imgs.append(dict(h=16, w=16, image_id=7, classes=np.array([79, 0, 5]), scores=np.array([0.5, 0.25, 0.7], np.float32),
                     boxes=np.array([[2, 2, 10, 10], [3, 5, 9, 5], [5, 5, 7, 7]], np.int64), masks=m))
    # a 1 x 1 image, set and unset
    imgs.append(dict(h=1, w=1, image_id=1000000007, classes=np.array([0, 79]),
                     scores=np.array([0.123456789, 0.987654321], np.float32),
                     boxes=np.array([[0, 0, 1, 1], [0, 0, 1, 1]], np.int64), masks=np.array([[[1]], [[0]]], np.uint8)))
    # YOLACT++ [box, mask] scores
    m = np.zeros((3, 20, 12), np.uint8)
    m[0, 2:18, 1:11] = 1
    m[1, :, 6:] = 1
    m[2, 10:, :] = 1
    imgs.append(dict(h=20, w=12, image_id=42, classes=np.array([12, 12, 60]),
                     scores=np.array([0.61, 0.6100001, 0.05], np.float32), boxes=np.array(
                         [[1, 2, 11, 18], [6, 0, 12, 20], [0, 10, 12, 20]], np.int64), masks=m,
                     mask_scores=np.array([0.3141592653589793, 0.7777777, 1e-7], np.float32)))
    return imgs


def random_images(r, count=6):
    imgs = []
    for j in range(count):
        h, w, n = int(r.randint(1, 70)), int(r.randint(1, 90)), int(r.randint(1, 12))
        x1, y1 = r.randint(0, w + 1, n), r.randint(0, h + 1, n)
        x2, y2 = np.minimum(x1 + r.randint(0, w, n), w), np.minimum(y1 + r.randint(0, h, n), h)
        boxes = np.stack([x1, y1, x2, y2], 1).astype(np.int64)
        masks = np.zeros((n, h, w), np.uint8)
        for i in range(n):
            masks[i, y1[i]:y2[i], x1[i]:x2[i]] = r.rand(y2[i] - y1[i], x2[i] - x1[i]) < 0.7
        img = dict(h=h, w=w, image_id=int(r.randint(0, 600000)), classes=r.randint(0, 80, n),
                   scores=r.rand(n).astype(np.float32), boxes=boxes, masks=masks)
        if j % 2:
            img["mask_scores"] = r.rand(n).astype(np.float32)
        imgs.append(img)
    return imgs


def main():
    from oracle import gen_golden as G
    from oracle.eval_oracle import rle_counts, rle_to_string
    G.install_shims()
    torch.Tensor.cuda = lambda self, *a, **k: self
    import pycocotools

    def encode(m):   # pycocotools.mask.encode of one Fortran-ordered [h, w] uint8 array
        return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": rle_to_string(rle_counts(m))}
    sys.modules["pycocotools.mask"].encode = encode
    pycocotools.mask = sys.modules["pycocotools.mask"]
    import eval as E
    from data.config import set_cfg
    set_cfg("yolact_base_config")
    tmp = tempfile.mkdtemp()
    bbox_file, mask_file = os.path.join(tmp, "bbox.json"), os.path.join(tmp, "mask.json")
    E.parse_args(["--output_coco_json", "--bbox_det_file=" + bbox_file, "--mask_det_file=" + mask_file, "--no_bar"])
    E.prep_coco_cats()
    detections = E.Detections()
    specs = crafted_images() + random_images(np.random.RandomState(2025))
    out = {"num_images": np.array(len(specs))}
    for i, a in enumerate(specs):
        h, w = a["h"], a["w"]
        cls, sc = torch.from_numpy(np.asarray(a["classes"], np.int64)), torch.from_numpy(a["scores"])
        scores = [sc, torch.from_numpy(a["mask_scores"])] if "mask_scores" in a else sc
        post = (cls, scores, torch.from_numpy(a["boxes"]), torch.from_numpy(a["masks"].astype(np.float32)))
        E.postprocess = lambda *args, _p=post, **kw: _p
        E.prep_metrics(None, None, None, None, None, h, w, 0, a["image_id"], detections)
        for key, v in a.items():
            v = np.packbits(v, axis=-1) if key == "masks" else np.asarray(v)
            out["img%d_%s" % (i, key)] = v
    detections.dump()
    keys = sorted(E.coco_cats)
    out["coco_cats_keys"] = np.array(keys, np.int64)
    out["coco_cats_values"] = np.array([E.coco_cats[k] for k in keys], np.int64)
    with open(bbox_file, "rb") as f:
        out["bbox_json"] = np.frombuffer(f.read(), np.uint8)
    with open(mask_file, "rb") as f:
        out["mask_json"] = np.frombuffer(f.read(), np.uint8)
    print("bbox records", len(detections.bbox_data), "mask records", len(detections.mask_data))
    G.npz_save("coco_json_unit", **out)


if __name__ == "__main__":
    main()
