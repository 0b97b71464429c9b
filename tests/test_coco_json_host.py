"""--output_coco_json's host side against tests/golden/coco_json_unit.npz (the real eval.py's records and JSON bytes): the
record builder, the golden's own RLE strings, and the GPU entry points' refusal of CPU tensors."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.eval_oracle import rle_counts, rle_decode, rle_from_string, rle_to_string
from yolact_b200 import _lib
from yolact_b200.metrics import Detections, append_coco_records

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "coco_json_unit.npz")


def golden():
    return np.load(GOLDEN)


def golden_images(z):
    ims = []
    for i in range(int(z["num_images"])):
        g = lambda key: z["img%d_%s" % (i, key)]
        h, w = int(g("h")), int(g("w"))
        im = dict(h=h, w=w, image_id=int(g("image_id")), classes=g("classes"), scores=g("scores"), boxes=g("boxes"),
                  masks=np.unpackbits(g("masks"), axis=-1, count=w).astype(np.uint8))
        ms = "img%d_mask_scores" % i
        im["mask_scores"] = z[ms] if ms in z.files else None
        ims.append(im)
    return ims


def category_table(z):
    table = [None] * (int(z["coco_cats_keys"].max()) + 1)
    for k, v in zip(z["coco_cats_keys"].tolist(), z["coco_cats_values"].tolist()):
        table[k] = v
    return table


def dumped(dets, tmp_path):
    b, m = tmp_path / "bbox.json", tmp_path / "mask.json"
    dets.dump(str(b), str(m))
    return b.read_bytes(), m.read_bytes()


@pytest.mark.parametrize("as_callable", [False, True])
def test_record_builder_reproduces_the_golden_json(tmp_path, as_callable):
    z = golden()
    table = category_table(z)
    dets = Detections((lambda c: table[c]) if as_callable else table)
    for im in golden_images(z):
        strings = [rle_to_string(rle_counts(m)).decode("ascii") for m in im["masks"]]
        ms = im["mask_scores"] if im["mask_scores"] is not None else im["scores"]
        append_coco_records(dets.bbox_data, dets.mask_data, dets.category_of, im["image_id"], im["classes"], im["boxes"],
                            im["scores"], ms, strings, im["h"], im["w"])
    bbox, mask = dumped(dets, tmp_path)
    assert bbox == z["bbox_json"].tobytes()
    assert mask == z["mask_json"].tobytes()
    # the zero-area boxes were skipped, and both lists stay paired
    assert len(dets.bbox_data) == len(dets.mask_data) < sum(len(im["classes"]) for im in golden_images(z))


def test_golden_covers_its_cases():
    z = golden()
    ims = golden_images(z)
    recs = json.loads(z["mask_json"].tobytes())
    counts = [rle_from_string(r["segmentation"]["counts"].encode()) for r in recs]
    assert any(c[0] == 0 for c in counts)                                     # a set first pixel
    assert any(len(c) == 1 for c in counts)                                   # an empty mask
    assert any(im["h"] == 1 and im["w"] == 1 for im in ims)
    cls = np.concatenate([im["classes"] for im in ims])
    assert 0 in cls and 79 in cls
    assert any(im["mask_scores"] is not None for im in ims)
    assert sorted(im["image_id"] for im in ims) != list(range(len(ims)))


def test_golden_strings_decode_to_the_stored_masks():
    z = golden()
    recs = iter(json.loads(z["mask_json"].tobytes()))
    for im in golden_images(z):
        b = im["boxes"]
        for i in np.flatnonzero((b[:, 3] - b[:, 1]) * (b[:, 2] - b[:, 0]) > 0):
            r = next(recs)
            assert r["segmentation"]["size"] == [im["h"], im["w"]]
            cnt = rle_from_string(r["segmentation"]["counts"].encode())
            assert (rle_decode(cnt, im["h"], im["w"]) == im["masks"][i]).all()


def test_entry_points_refuse_cpu_tensors():
    det = {"box": torch.zeros(1, 4), "mask": torch.zeros(1, 32), "class": torch.zeros(1, dtype=torch.int64),
           "score": torch.ones(1), "proto": torch.zeros(4, 4, 32)}
    with pytest.raises(_lib.YbError, match="no CPU path"):
        Detections(list(range(80))).add([{"net": None, "detection": det}], [(8, 8)], [0])
