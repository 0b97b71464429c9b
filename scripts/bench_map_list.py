"""Time per image of eval.py's mAP bookkeeping (prep_metrics, eval.py:386-510) over 64 COCO-sized frames, two routes:

  (a) metrics.prep_metrics per image: postprocess(mask_format='bits') writes every mask, the ground truth goes up in
      three pinned copies, two jaccard, two mask_iou and one yb_eval_match launch;
  (b) metrics.prep_metrics_list per list of 8 images: postprocess_list without masks, the ground truth of the list in
      one pinned buffer and one H2D copy, one pack launch, one yb_eval_iou_list and one yb_eval_match_list launch.

yolact_base at 550 with the deterministic weights (oracle/weights.py) through forward_frames in lists of 8, on seeded
uint8 BGR frames of the 16 sizes of bench_frame_list.py, four times over (score_threshold 0).  Each image gets seeded
synthetic ground truth: 7 objects and 1 crowd whose masks spill past their boxes, in the dataset's form (host fp32).
Both routes run once to warm up and once counted (launches of the ops handles, host syncs as torch's sync-debug mode
reports them), then --rounds rounds alternate the two routes; the table gives the median host wall ms per image (host
clock around the route and a device synchronise) and the median CUDA-event ms per image over the same window.  The
two routes' raw records, counts and calc_map all_maps must be identical.  Prints the GPU name and power limit, which
belong with every number.

    python scripts/bench_map_list.py [--rounds 5]
"""
import argparse
import os
import statistics
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import yolact_b200
from bench_frame_list import SIZES, gpu_info
from oracle.weights import deterministic_state_dict
from yolact_b200.config import CONFIGS
from yolact_b200.metrics import APData, calc_map, prep_metrics, prep_metrics_list
from yolact_b200.output_utils import launch_count

LIST = 8


def ground_truth(preds, sizes, seed):
    """7 objects (about half of them over a detection of its class) and 1 crowd per image, masks spilling past the
    boxes."""
    r = np.random.RandomState(seed)
    gts, gms, ncs = [], [], []
    for p, (h, w) in zip(preds, sizes):
        g, nc = 7, 1
        gt = np.zeros((g + nc, 5), np.float32)
        c, wh = r.uniform(0, 1, (g + nc, 2)), r.uniform(0.05, 0.6, (g + nc, 2))
        gt[:, :2], gt[:, 2:4] = c - wh / 2, c + wh / 2
        gt[:, 4] = r.randint(0, 80, g + nc)
        det = p["detection"]
        if det is not None:
            k = min(4, int(det["box"].shape[0]))
            gt[:k, :4] = det["box"][:k].cpu().numpy() + r.uniform(-0.02, 0.02, (k, 4))
            gt[:k, 4] = det["class"][:k].cpu().numpy()
        gm = np.zeros((g + nc, h, w), np.float32)
        for j in range(g + nc):
            x1, y1, x2, y2 = gt[j, :4]
            ex = r.uniform(0.01, 0.08)
            ys = slice(max(0, int((y1 - ex) * h)), max(1, int(np.ceil((y2 + ex) * h))))
            xs = slice(max(0, int((x1 - ex) * w)), max(1, int(np.ceil((x2 + ex) * w))))
            gm[j, ys, xs] = 1
        gts.append(gt)
        gms.append(gm)
        ncs.append(nc)
    return gts, gms, ncs


def route_a(preds, sizes, gts, gms, ncs):
    apd = APData(80)
    for i, (h, w) in enumerate(sizes):
        prep_metrics(apd, preds[i:i + 1], None, gts[i], gms[i], h, w, ncs[i], i)
    return apd


def route_b(preds, sizes, gts, gms, ncs):
    apd = APData(80)
    for s in range(0, len(preds), LIST):
        sl = slice(s, s + LIST)
        prep_metrics_list(apd, preds[sl], sizes[sl], gts[sl], gms[sl], ncs[sl])
    return apd


def counted(fn):
    """-> (result, launches, host syncs) of one run of fn."""
    torch.cuda.synchronize()
    n0 = launch_count()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    syncs = sum("synchroniz" in str(w.message) for w in caught)
    return out, launch_count() - n0, syncs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print("GPU:", gpu_info())
    cfg = CONFIGS["yolact_base_config"].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision="f16x3")
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    sizes = SIZES * 4
    preds = []
    for s in range(0, len(sizes), LIST):
        g = torch.Generator().manual_seed(s)
        preds += net.forward_frames([torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda()
                                     for h, w in sizes[s:s + LIST]])
    gts, gms, ncs = ground_truth(preds, sizes, 17)
    N = len(preds)
    ns = [0 if p["detection"] is None else int(p["detection"]["box"].shape[0]) for p in preds]
    routes = {"(a) prep_metrics, per image": route_a, "(b) prep_metrics_list, per list of 8": route_b}
    res, stats = {}, {}
    for name, fn in routes.items():
        fn(preds, sizes, gts, gms, ncs)   # warm-up
        apd, launches, syncs = counted(lambda: fn(preds, sizes, gts, gms, ncs))
        score, tag = apd._host_records()
        res[name] = (score.view(np.uint32), tag, apd.num_gt_positives(), calc_map(apd, print_table=False))
        stats[name] = (launches / N, syncs / N)
    wall, dev = {k: [] for k in routes}, {k: [] for k in routes}
    for _ in range(args.rounds):   # the routes alternate within each round
        for name, fn in routes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            fn(preds, sizes, gts, gms, ncs)
            e1.record()
            torch.cuda.synchronize()
            wall[name].append((time.perf_counter() - t0) * 1e3 / N)
            dev[name].append(e0.elapsed_time(e1) / N)
    a, b = (res[k] for k in routes)
    same_records = all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3]))
    same_maps = a[3] == b[3]
    print("%d images, %d..%d detections each, %d records" % (N, min(ns), max(ns), len(a[1])))
    print("| route | host wall ms / image | CUDA-event ms / image | launches / image | host syncs / image |")
    print("|---|---|---|---|---|")
    for name in routes:
        la, sy = stats[name]
        print("| %s | %.3f | %.3f | %.2f | %.2f |" % (name, statistics.median(wall[name]), statistics.median(dev[name]),
                                                    la, sy))
    print("records identical: %s, all_maps identical: %s" % (same_records, same_maps))
    print("all_maps:", a[3])
    assert same_records and same_maps, "the two routes differ"


if __name__ == "__main__":
    main()
