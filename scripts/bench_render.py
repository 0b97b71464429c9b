"""Time per frame of prep_display's GPU part (undo_transform=False, no text or boxes) for a list of 8 frames per call:

  (a) the composition a caller runs today, per image: postprocess with rescore_bbox (masks at frame size for all n
      detections, fp32 or uint8), argsort, a gather of the top_k masks, .cpu() of classes / scores / boxes, display_blend;
  (b) render_masks on the whole list: one selection launch and one render launch, no masks written.

yolact_base detections (n = 100 per image, deterministic weights through forward_frames at 550^2) on seeded uint8 BGR
frames of 550x550, 480x640 and 1080x1920, top_k 5 and 15, score_threshold 0.  The paths alternate, one window each per
round, every window ending in a device synchronise; the table gives the median over rounds as CUDA-event ms per frame
and host wall ms per frame, the kernel launches per call of 8 frames (the ops handle's counter), and whether (a) and (b)
give identical images.  Prints the GPU name and power limit, which belong with every number.

    python scripts/bench_render.py [--rounds 5]
"""
import argparse
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import yolact_b200
from bench_frame_list import gpu_info
from oracle.weights import deterministic_state_dict
from yolact_b200 import config as ybcfg
from yolact_b200.config import CONFIGS
from yolact_b200.display import render_masks
from yolact_b200.eval_utils import display_blend, get_color
from yolact_b200.output_utils import launch_count, postprocess


def composition(preds, frames, top_k, fmt):
    cfg = ybcfg.cfg
    out = []
    for i, f in enumerate(frames):
        save, cfg.rescore_bbox = cfg.rescore_bbox, True
        try:
            t = postprocess(preds, int(f.shape[1]), int(f.shape[0]), i, mask_format=fmt)
        finally:
            cfg.rescore_bbox = save
        idx = t[1].argsort(0, descending=True)[:top_k]
        masks = t[3][idx]
        classes, scores, boxes = t[0][idx].cpu().numpy(), t[1][idx].cpu().numpy(), t[2][idx].cpu().numpy()
        n = min(top_k, classes.shape[0])
        colors = [[c / 255.0 for c in get_color(j, classes, False, bgr=True)] for j in range(n)]
        out.append(display_blend(f.float(), masks[:n] if n else None, colors if n else None, 0.45))
    return out


def window(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3, out


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
    B = 8
    print("| frames | top_k | path | event ms / frame | wall ms / frame | launches / call | identical |")
    print("|---|---|---|---|---|---|---|")
    for (h, w) in ((550, 550), (480, 640), (1080, 1920)):
        g = torch.Generator().manual_seed(h * w)
        frames = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for _ in range(B)]
        preds = net.forward_frames(frames)
        ns = [0 if p["detection"] is None else int(p["detection"]["box"].shape[0]) for p in preds]
        for top_k in (5, 15):
            paths = {"(a) composition, f32 masks": lambda: composition(preds, frames, top_k, "f32"),
                     "(a) composition, u8 masks": lambda: composition(preds, frames, top_k, "u8"),
                     "(b) render_masks": lambda: render_masks(preds, frames, top_k=top_k)[0]}
            results, launches, times = {}, {}, {k: [] for k in paths}
            for name, fn in paths.items():   # warm-up, launch count and the images
                fn()
                n0 = launch_count()
                results[name] = window(fn)[2]
                launches[name] = launch_count() - n0
            for _ in range(args.rounds):
                for name, fn in paths.items():
                    ev, wall, _ = window(fn)
                    times[name].append((ev / B, wall / B))
            ref = results["(b) render_masks"]
            for name in paths:
                same = all(torch.equal(a, b) for a, b in zip(results[name], ref))
                ev = statistics.median(t[0] for t in times[name])
                wall = statistics.median(t[1] for t in times[name])
                print("| %dx%d (n %d..%d) | %d | %s | %.3f | %.3f | %d | %s |" % (h, w, min(ns), max(ns), top_k, name, ev,
                                                                              wall, launches[name], same))


if __name__ == "__main__":
    main()
