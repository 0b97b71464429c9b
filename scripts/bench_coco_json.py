"""Host wall time per image of eval.py's --output_coco_json records (prep_metrics' JSON branch, eval.py:414-429) over 64
COCO-sized frames, three routes:

  (a) today's best composition, per image: postprocess(mask_format='bits') + eval_utils.encode_masks (yb_mask_rle, a
      host sync, the capped run buffer to the host, rle_to_string per row) + the records;
  (b) metrics.Detections.add per image: yb_postprocess_list without masks, one yb_coco_rle_list launch, one D2H copy;
  (c) metrics.Detections.add per list of 8 images.

yolact_base at 550 with the deterministic weights (oracle/weights.py) through forward_frames on seeded uint8 BGR frames
of the 16 sizes of bench_frame_list.py, four times over (100 detections per image, score_threshold 0).  Each route runs
once to warm up, then --rounds times over all 64 frames; the table gives the median host wall ms per image (every route
ends in host records, so wall time is the cost), kernel launches per image (the ops handle's counter), host syncs and
D2H bytes per image (counted at Tensor.cpu, the only way either route brings data to the host).  The three routes' dump
bytes must be identical.  Prints the GPU name and power limit, which belong with every number.

    python scripts/bench_coco_json.py [--rounds 3]
"""
import argparse
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import yolact_b200
from bench_frame_list import SIZES, gpu_info
from oracle.weights import deterministic_state_dict
from yolact_b200.config import CONFIGS
from yolact_b200.eval_utils import encode_masks
from yolact_b200.metrics import Detections, append_coco_records
from yolact_b200.output_utils import launch_count, postprocess

CATS = list(range(1, 81))
D2H = {"copies": 0, "bytes": 0}
_cpu = torch.Tensor.cpu


def counting_cpu(self, *a, **k):
    if self.is_cuda:
        D2H["copies"] += 1
        D2H["bytes"] += self.numel() * self.element_size()
    return _cpu(self, *a, **k)


def route_a(preds, sizes, ids):
    dets = Detections(CATS)
    for i, ((h, w), image_id) in enumerate(zip(sizes, ids)):
        classes, scores, boxes, masks = postprocess(preds, w, h, i, mask_format="bits")
        if classes.size(0) == 0:
            continue
        bs, ms = (scores[0], scores[1]) if isinstance(scores, list) else (scores, scores)
        counts = [e["counts"].decode("ascii") for e in encode_masks(masks, "bits", w)]
        append_coco_records(dets.bbox_data, dets.mask_data, CATS, image_id, classes.cpu().numpy(), boxes.cpu().numpy(),
                            bs.cpu().numpy(), ms.cpu().numpy(), counts, h, w)
    return dets


def route_add(preds, sizes, ids, per_call):
    dets = Detections(CATS)
    for s in range(0, len(preds), per_call):
        dets.add(preds[s:s + per_call], sizes[s:s + per_call], ids[s:s + per_call])
    return dets


def dump_bytes(dets):
    d = tempfile.mkdtemp()
    b, m = os.path.join(d, "b.json"), os.path.join(d, "m.json")
    dets.dump(b, m)
    return open(b, "rb").read() + b"|" + open(m, "rb").read()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    sizes = SIZES * 4
    preds = []
    for s in range(0, len(sizes), 8):
        g = torch.Generator().manual_seed(s)
        preds += net.forward_frames([torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda()
                                     for h, w in sizes[s:s + 8]])
    ns = [0 if p["detection"] is None else int(p["detection"]["box"].shape[0]) for p in preds]
    ids = [1000 + 7 * i for i in range(len(preds))]
    N = len(preds)
    routes = {"(a) postprocess bits + encode_masks, per image": lambda: route_a(preds, sizes, ids),
              "(b) Detections.add, per image": lambda: route_add(preds, sizes, ids, 1),
              "(c) Detections.add, per list of 8": lambda: route_add(preds, sizes, ids, 8)}
    dumps, stats, times = {}, {}, {k: [] for k in routes}
    torch.Tensor.cpu = counting_cpu
    try:
        for name, fn in routes.items():   # warm-up, then one counted run
            fn()
            torch.cuda.synchronize()
            D2H["copies"] = D2H["bytes"] = 0
            n0 = launch_count()
            dumps[name] = dump_bytes(fn())
            torch.cuda.synchronize()
            stats[name] = ((launch_count() - n0) / N, D2H["copies"] / N, D2H["bytes"] / N)
    finally:
        torch.Tensor.cpu = _cpu
    for _ in range(args.rounds):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / N)
    ref = dumps["(a) postprocess bits + encode_masks, per image"]
    print("%d images, %d..%d detections each, %d mask records" % (N, min(ns), max(ns), ref.count(b'"segmentation"')))
    print("| route | host wall ms / image | launches / image | host syncs / image | D2H bytes / image | dump identical |")
    print("|---|---|---|---|---|---|")
    for name in routes:
        la, sy, by = stats[name]
        print("| %s | %.3f | %.2f | %.2f | %.0f | %s |" % (name, statistics.median(times[name]), la, sy, by,
                                                         dumps[name] == ref))
    assert all(d == ref for d in dumps.values()), "the routes' dump bytes differ"


if __name__ == "__main__":
    main()
