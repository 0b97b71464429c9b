"""Time per image of postprocessing a folder of differently sized images (COCO-like sizes), two ways:

  (a) postprocess(preds, w_i, h_i, i) per image: one yb_postprocess call (2 launches, 10 with YOLACT++'s maskiou) and,
      with score_threshold > 0, one host sync per image;
  (b) postprocess_list(preds, sizes) per batch: one call and one launch per kernel for the whole batch.

yolact_base (and one yolact_plus_base row) at 550^2 with deterministic weights (100 detections per image); 64 seeded
uint8 BGR frames cycle through 16 sizes, batch 8.  forward_frames runs once per batch, outside the timed windows; every
window postprocesses copies of those detections (the threshold filters them in place), made before the window.  The
paths are alternated, one window (all 64 images) each per round, every window ending in a device synchronise; the table
gives the median over rounds and the range, as CUDA-event time and host wall time (the saving is partly host-side).
Prints the GPU name and power limit, which belong with every number, and whether (a) and (b) are bit-identical.

    python scripts/bench_postprocess_list.py [--precision f16x3] [--rounds 5] [--batch 8]
"""
import argparse
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import yolact_b200
from bench_frame_list import SIZES, gpu_info
from oracle.weights import deterministic_state_dict
from yolact_b200.config import CONFIGS
from yolact_b200.output_utils import postprocess, postprocess_list


def clone(preds):
    return [{"detection": None if p["detection"] is None else dict(p["detection"]), "net": p["net"]} for p in preds]


def window(fn):
    """(CUDA-event ms, host wall ms) of fn(), from a synchronised device to a synchronised device."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    del out
    return e0.elapsed_time(e1), (t1 - t0) * 1e3


def identical(a, b):
    for x, y in zip(a, b):
        if isinstance(x, list):
            if not identical(x, y):
                return False
        elif x.dtype != y.dtype or x.shape != y.shape or not torch.equal(x, y):
            return False
    return True


def make(config, precision):
    cfg = CONFIGS[config].copy()
    yolact_b200.cfg.replace(cfg.copy())
    net = yolact_b200.Yolact(cfg, precision=precision)
    net.detect.use_fast_nms = True
    net.load_state_dict(deterministic_state_dict(net.state_dict(), 0))
    net.eval()
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16x3", choices=["f16x3", "f16tc", "f32"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--images", type=int, default=64)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_postprocess_list measures on the GPU; there is no CPU fallback"
    assert a.images % a.batch == 0
    rng = np.random.RandomState(0)
    frames = [torch.from_numpy(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)).cuda()
              for h, w in (SIZES[i % len(SIZES)] for i in range(a.images))]
    batches = [frames[i:i + a.batch] for i in range(0, a.images, a.batch)]
    sizes = [[tuple(f.shape[:2]) for f in fs] for fs in batches]

    rows = [("yolact_base", "f32", 0), ("yolact_base", "bits", 0), ("yolact_base", "f32", 0.15),
            ("yolact_base", "bits", 0.15), ("yolact_plus_base", "bits", 0)]
    nets, preds = {}, {}
    print("# %s; %s @550, %d uint8 BGR frames cycling through %d sizes, batch %d; median of %d alternated windows "
          "(range)" % (gpu_info(), a.precision, a.images, len(SIZES), a.batch, a.rounds))
    print("| model | mask_format | score_threshold | dets / image | (a) per image: event ms / image | (a) wall | "
          "(b) list: event ms / image | (b) wall | (b)/(a) event | (b)/(a) wall | identical |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for model, fmt, thr in rows:
        if model not in nets:
            nets[model] = make(model + "_config", a.precision)
            preds[model] = [nets[model].forward_frames(fs) for fs in batches]
        net, P = nets[model], preds[model]
        yolact_b200.cfg.replace(net.cfg.copy())
        torch.cuda.synchronize()
        ndet = statistics.mean(0 if p["detection"] is None else int(p["detection"]["score"].shape[0])
                               for ps in P for p in ps)

        def loop(copies):
            return [[postprocess(ps, w, h, i, score_threshold=thr, mask_format=fmt)
                     for i, (h, w) in enumerate(sz)] for ps, sz in zip(copies, sizes)]

        def lists(copies):
            return [postprocess_list(ps, sz, score_threshold=thr, mask_format=fmt) for ps, sz in zip(copies, sizes)]

        paths = [loop, lists]
        for fn in paths:   # warm-up: handles, item table, allocator
            fn([clone(ps) for ps in P])
        ra, rb = loop([clone(ps) for ps in P]), lists([clone(ps) for ps in P])
        torch.cuda.synchronize()
        same = all(identical(x, y) for ba, bb in zip(ra, rb) for x, y in zip(ba, bb))
        del ra, rb
        ev = [[] for _ in paths]
        wall = [[] for _ in paths]
        for _ in range(a.rounds):
            for e, w, fn in zip(ev, wall, paths):
                copies = [clone(ps) for ps in P]
                te, tw = window(lambda: fn(copies))
                e.append(te / a.images)
                w.append(tw / a.images)

        def cell(t):
            return "%.3f (%.3f-%.3f)" % (statistics.median(t), min(t), max(t))

        print("| %s | %s | %g | %.0f | %s | %s | %s | %s | %.2f | %.2f | %s |" % (
            model, fmt, thr, ndet, cell(ev[0]), cell(wall[0]), cell(ev[1]), cell(wall[1]),
            statistics.median(ev[1]) / statistics.median(ev[0]), statistics.median(wall[1]) / statistics.median(wall[0]),
            same), flush=True)


if __name__ == "__main__":
    main()
